"""SDXL T2I-Adapter ([3P] diffusers 0.30.0 `T2IAdapter` with adapter_type "full_adapter_xl", and `MultiAdapter`) on the
sm_90a kernel library.  Restated from the published diffusers sources, parity unpinned (no diffusers output is pinned
by a golden here).  Module tree and state-dict keys are diffusers':

    adapter.conv_in                                3x3, in_channels * 256 -> channels[0]
    adapter.body.{i}.in_conv                       1x1, channels[i-1] -> channels[i]   (blocks 1 and 2 only)
    adapter.body.{i}.resnets.{j}.block1 / block2   3x3 / 1x1, channels[i] -> channels[i]

    forward(x):  x = PixelUnshuffle(16)(x); x = conv_in(x)
                 block 0:           resnets
                 block 1:           in_conv, resnets
                 block 2:           AvgPool2d(2, ceil_mode=True), in_conv, resnets
                 block 3:           resnets
                 resnet(x) = block2(relu(block1(x))) + x;   returns the 4 block outputs

At 1024^2 the features are 320@64^2, 640@64^2, 1280@32^2 and 1280@32^2: the UNet adds them inside its encoder
(UNet2DConditionModel.forward(adapter_residuals=), diffusers' down_intrablock_additional_residuals).

Every layer runs on existing kernels of this package, activations NHWC fp16:

* PixelUnshuffle(16): a torch reshape/permute of the [B, C, H, W] image into NHWC [B, H/16, W/16, 256 C] with
  diffusers' channel order c * 256 + i * 16 + j; layout plumbing done once per call, like the control-image
  preprocessing of the ControlNet pipeline;
* conv_in and every block1: the implicit-GEMM 3x3 conv, block1 with the ReLU epilogue (IH_EPI_RELU);
* block2 + the skip, and block 1's in_conv: the GEMM (ops.linear), block2 with the skip as its residual operand;
* block 2's AvgPool2d(2) + 1x1 in_conv: ONE 2x2-window, stride-2 conv on ih_conv2d_down_f16 (ops.conv3x3_down, a 3x3
  stride-2 conv of the bottom/right-padded input) whose 3x3 weight holds w / 4 at taps (0, 0), (0, 1), (1, 0), (1, 1)
  and zeros at the others; the padding row and column are only read by the zero taps.  pool-then-conv equals this
  in real arithmetic, but diffusers rounds the pooled activations to fp16 and the fold does not: it rounds once where
  diffusers rounds twice (about one fp16 ulp of the output apart); a w / 4 below the fp16 normal range (|w| < 2^-12)
  is rounded to the subnormal grid, off by at most 2^-25.  `ceil_mode` never applies: every SDXL size gives an
  even 64^2 / 32^2-style grid, and an odd grid (image sides not multiples of 32) raises IHError.

Deviations from diffusers, written down: only `full_adapter_xl` is built; the SD1.5 types `full_adapter` and
`light_adapter` and any other `num_res_blocks` / `downscale_factor` raise IHError.  `channels` must have the XL
pattern (c, 2c, 4c, 4c) with c a multiple of 64 (SDXL's (320, 640, 1280, 1280); the tests' miniature (64, 128, 256,
256)).  MultiAdapter keeps diffusers' sum -- feature k = fp16(w_0 f_0k), then acc = fp16(acc + fp16(w_j f_jk)) in
adapter order, the weights fp32 -- but computes it with one ih_controlnet_add_residuals_multi_f16 launch into a zeroed
buffer (the kernel's skip + acc with skip = 0 is acc; a -0.0 sum comes out +0.0).  With a MultiAdapter the pipeline
takes a float adapter_conditioning_scale (the default 1.0 included) as the weight of every adapter; diffusers'
MultiAdapter fails on a float (torch.tensor(float) is 0-d and cannot be zipped), so there only a list works.  The
pipeline's default height and width are the image's rounded down to a multiple of the downscale factor (16) as in
diffusers, not of 32; a size that is an odd multiple of 16 is then refused (IHError), as the UNet would refuse it.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

from . import ops
from ._lib import IH_CN_MAX_NETS, IHError
from .config import SDXL_T2I_ADAPTER, T2IAdapterConfig


def check_config(cfg: T2IAdapterConfig) -> T2IAdapterConfig:
    """IHError for every T2IAdapter configuration the native adapter does not implement (see the module docstring)."""
    if cfg.adapter_type in ("full_adapter", "light_adapter"):
        raise IHError(f"T2IAdapter: adapter_type {cfg.adapter_type!r} (the SD1.5 architectures) is not implemented; "
                      "only 'full_adapter_xl' is")
    if cfg.adapter_type != "full_adapter_xl":
        raise IHError(f"T2IAdapter: unknown adapter_type {cfg.adapter_type!r}")
    c = tuple(int(x) for x in cfg.channels)
    if len(c) != 4 or c[0] <= 0 or c[0] % 64 or c != (c[0], 2 * c[0], 4 * c[0], 4 * c[0]):
        raise IHError(f"T2IAdapter: channels {list(c)} are not implemented: full_adapter_xl needs (c, 2c, 4c, 4c) with c "
                      "a multiple of 64, e.g. [320, 640, 1280, 1280]")
    if cfg.num_res_blocks != 2:
        raise IHError(f"T2IAdapter: num_res_blocks = {cfg.num_res_blocks} is not implemented (only 2)")
    if cfg.downscale_factor != 16:
        raise IHError(f"T2IAdapter: downscale_factor = {cfg.downscale_factor} is not implemented (only 16, the XL "
                      "adapters')")
    if cfg.in_channels not in (1, 3):
        raise IHError(f"T2IAdapter: in_channels = {cfg.in_channels} is not implemented (1 or 3)")
    return cfg


def config_from_diffusers(meta: dict) -> T2IAdapterConfig:
    """A diffusers T2IAdapter config.json (as a dict) -> T2IAdapterConfig, refused (IHError) as in check_config.
    diffusers' own defaults apply to absent fields (adapter_type "full_adapter", downscale_factor 8)."""
    cfg = T2IAdapterConfig(in_channels=int(meta.get("in_channels", 3)),
                           channels=tuple(int(c) for c in meta.get("channels", (320, 640, 1280, 1280))),
                           num_res_blocks=int(meta.get("num_res_blocks", 2)),
                           downscale_factor=int(meta.get("downscale_factor", 8)),
                           adapter_type=str(meta.get("adapter_type", "full_adapter")))
    return check_config(cfg)


class AdapterResnetBlock(nn.Module):
    def __init__(self, ch: int):
        super().__init__()
        self.block1 = nn.Conv2d(ch, ch, 3, padding=1)
        self.block2 = nn.Conv2d(ch, ch, 1)
        self._w1 = self._w2 = None

    def finalize(self):
        self._w1 = ops.pack_conv3x3_weight(self.block1.weight.detach())
        self._w2 = self.block2.weight.detach().reshape(self.block2.weight.shape[0], -1).contiguous()

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        B, H, W, C = x.shape
        h = ops.conv3x3(x, self._w1, self.block1.bias, relu=True)                  # relu(block1(x))
        y = ops.linear(h.reshape(B * H * W, C), self._w2, self.block2.bias, residual=x.reshape(B * H * W, C))
        return y.reshape(B, H, W, C)                                               # block2(.) + x


class AdapterBlock(nn.Module):
    def __init__(self, cin: int, cout: int, num_res_blocks: int, down: bool = False):
        super().__init__()
        self.down = down
        self.in_conv = nn.Conv2d(cin, cout, 1) if cin != cout else None
        if down and self.in_conv is None:
            raise IHError("T2IAdapter: the downsampling block needs an in_conv to fold the average pool into")
        self.resnets = nn.Sequential(*[AdapterResnetBlock(cout) for _ in range(num_res_blocks)])
        self._w_in = None

    def finalize(self):
        for r in self.resnets:
            r.finalize()
        if self.in_conv is None:
            return
        w = self.in_conv.weight.detach()                                           # [cout, cin, 1, 1]
        if self.down:          # AvgPool2d(2) then the 1x1 conv: one 2x2 window conv, w / 4 at the top-left 2x2 taps
            w3 = torch.zeros((w.shape[0], w.shape[1], 3, 3), dtype=w.dtype, device=w.device)
            w3[:, :, :2, :2] = (w.float() / 4).to(w.dtype)         # exact unless w / 4 is subnormal (module docstring)
            self._w_in = ops.pack_conv3x3_weight(w3)
        else:
            self._w_in = w.reshape(w.shape[0], w.shape[1]).contiguous()

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.in_conv is not None:
            B, H, W, C = x.shape
            if self.down:
                x = ops.conv3x3_down(x, self._w_in, self.in_conv.bias)
            else:
                x = ops.linear(x.reshape(B * H * W, C), self._w_in, self.in_conv.bias).reshape(B, H, W, -1)
        for r in self.resnets:
            x = r(x)
        return x


class FullAdapterXL(nn.Module):
    def __init__(self, cfg: T2IAdapterConfig):
        super().__init__()
        c = cfg.channels
        self.downscale_factor = cfg.downscale_factor
        self.conv_in = nn.Conv2d(cfg.in_channels * cfg.downscale_factor ** 2, c[0], 3, padding=1)
        self.body = nn.ModuleList([AdapterBlock(c[0], c[0], cfg.num_res_blocks),
                                   AdapterBlock(c[0], c[1], cfg.num_res_blocks),
                                   AdapterBlock(c[1], c[2], cfg.num_res_blocks, down=True),
                                   AdapterBlock(c[2], c[3], cfg.num_res_blocks)])


def pixel_unshuffle_nhwc(x: torch.Tensor, r: int) -> torch.Tensor:
    """[3P] torch.nn.PixelUnshuffle(r) followed by NCHW -> NHWC: [B, C, H, W] -> [B, H/r, W/r, C r^2], output channel
    c * r^2 + i * r + j holding x[b, c, y * r + i, x * r + j]."""
    B, C, H, W = x.shape
    return x.reshape(B, C, H // r, r, W // r, r).permute(0, 2, 4, 1, 3, 5).reshape(B, H // r, W // r, C * r * r)


def require_image_size(cfg: T2IAdapterConfig, height: int, width: int) -> None:
    """IHError unless a height x width image unshuffles into an even grid (the average pool of block 2 then never
    needs ceil_mode): both sides multiples of 2 * downscale_factor = 32 pixels, as every SDXL size is."""
    m = 2 * cfg.downscale_factor
    if height % m or width % m:
        raise IHError(f"T2IAdapter: image size {height}x{width} is not supported: the sides must be multiples of {m} "
                      f"pixels (an even {cfg.downscale_factor}x-unshuffled grid for the 2x2 average pool)")


class T2IAdapter(nn.Module):
    """Native SDXL T2I-Adapter.  Build with `from_pretrained`, `from_state_dict` or `from_random`."""

    def __init__(self, cfg: T2IAdapterConfig = SDXL_T2I_ADAPTER):
        super().__init__()
        self.config = check_config(cfg)
        self.adapter = FullAdapterXL(cfg)
        self._w_in = None
        self.graph_epoch = 0

    @property
    def downscale_factor(self) -> int:
        return self.config.downscale_factor

    @property
    def total_downscale_factor(self) -> int:
        return 2 * self.config.downscale_factor              # [3P] FullAdapterXL: one downsampling block

    # ---- construction ------------------------------------------------------------------------------------------
    @classmethod
    def from_state_dict(cls, cfg: T2IAdapterConfig, sd, device="cuda") -> "T2IAdapter":
        """`sd` must hold exactly the keys and shapes `cfg` builds (diffusers' names)."""
        with torch.device("meta"):
            m = cls(cfg)
        own = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        have = {k: tuple(v.shape) for k, v in sd.items()}
        missing, extra = sorted(set(own) - set(have)), sorted(set(have) - set(own))
        shapes = sorted(k for k in set(own) & set(have) if own[k] != have[k])
        if missing or extra or shapes:
            raise IHError(f"T2IAdapter: the checkpoint does not match channels {list(cfg.channels)} / in_channels "
                          f"{cfg.in_channels}: missing {missing[:3]}, unexpected {extra[:3]}, other shapes {shapes[:3]}")
        m = m.to_empty(device=device)
        m.load_state_dict({k: sd[k].to(device=device, dtype=torch.float16) for k in own})
        m = m.half().eval().requires_grad_(False)
        m.finalize()
        return m

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=torch.float16, device="cuda", **kwargs) -> "T2IAdapter":
        """A diffusers T2IAdapter folder (e.g. TencentARC/t2i-adapter-sketch-sdxl-1.0): config.json +
        diffusion_pytorch_model[.fp16].safetensors or diffusion_pytorch_model.bin."""
        if torch_dtype != torch.float16:
            raise IHError(f"T2IAdapter runs in fp16 (torch_dtype={torch_dtype} requested)")
        with open(os.path.join(path, "config.json")) as f:
            cfg = config_from_diffusers(json.load(f))
        for name in ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors"):
            f = os.path.join(path, name)
            if os.path.exists(f):
                from safetensors.torch import load_file
                return cls.from_state_dict(cfg, load_file(f), device=device)
        f = os.path.join(path, "diffusion_pytorch_model.bin")
        if os.path.exists(f):
            return cls.from_state_dict(cfg, torch.load(f, map_location="cpu", weights_only=True), device=device)
        raise FileNotFoundError(f"no T2IAdapter weights (diffusion_pytorch_model[.fp16].safetensors / .bin) under {path}")

    @classmethod
    def from_random(cls, cfg: T2IAdapterConfig = SDXL_T2I_ADAPTER, seed: int = 0, device="cuda") -> "T2IAdapter":
        """Random-init weights of the architecture (benchmarks and tests)."""
        from .weights import random_state_dict, shapes_of
        with torch.device("meta"):
            shapes = shapes_of(cls(cfg))
        return cls.from_state_dict(cfg, random_state_dict(shapes, seed, device=device), device=device)

    def finalize(self) -> None:
        """Derive the kernel-layout weights.  Call after (re)loading parameters."""
        for blk in self.adapter.body:
            blk.finalize()
        self._w_in = ops.pack_conv3x3_weight(self.adapter.conv_in.weight.detach())
        self.graph_epoch += 1

    # ---- forward -----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        """x: the adapter image NCHW [B, in_channels, H, W] (fp16, values in [0, 1]) -> the 4 features NHWC fp16
        [B, H/16, W/16, c0], [B, H/16, W/16, c1], [B, H/32, W/32, c2], [B, H/32, W/32, c3]."""
        if self._w_in is None:
            raise IHError("T2IAdapter.finalize() has not run (use from_pretrained / from_state_dict / from_random)")
        cfg = self.config
        if x.dim() != 4 or x.shape[1] != cfg.in_channels:
            raise IHError(f"T2IAdapter: expected an image [B, {cfg.in_channels}, H, W], got {tuple(x.shape)}")
        require_image_size(cfg, x.shape[2], x.shape[3])
        h = pixel_unshuffle_nhwc(x.to(self._w_in.dtype), cfg.downscale_factor).contiguous()
        h = ops.conv3x3(h, self._w_in, self.adapter.conv_in.bias)
        feats = []
        for blk in self.adapter.body:
            h = blk(h)
            feats.append(h)
        return feats


class MultiAdapter(nn.Module):
    """[3P] diffusers MultiAdapter: several T2IAdapters (`.adapters`, 2 .. 8) whose features are summed with per-adapter
    weights.  All of them must share `channels` and the downscale factor."""

    def __init__(self, adapters: Sequence[T2IAdapter]):
        super().__init__()
        adapters = list(adapters)
        if len(adapters) < 2:
            raise IHError(f"MultiAdapter: {len(adapters)} adapters; use a T2IAdapter for one")
        if len(adapters) > IH_CN_MAX_NETS:
            raise IHError(f"MultiAdapter: {len(adapters)} adapters, at most {IH_CN_MAX_NETS} are supported")
        for i, a in enumerate(adapters):
            if not isinstance(a, T2IAdapter):
                raise IHError(f"MultiAdapter: entry {i} is {type(a).__name__}, not a T2IAdapter")
            c0, ci = adapters[0].config, a.config
            if tuple(ci.channels) != tuple(c0.channels) or ci.downscale_factor != c0.downscale_factor:
                raise IHError(f"MultiAdapter: adapter {i} has channels {list(ci.channels)} / downscale factor "
                              f"{ci.downscale_factor}, adapter 0 has {list(c0.channels)} / {c0.downscale_factor}")
        self.adapters = nn.ModuleList(adapters)
        self.num_adapter = len(adapters)
        self.config = adapters[0].config

    @property
    def downscale_factor(self) -> int:
        return self.config.downscale_factor

    @property
    def total_downscale_factor(self) -> int:
        return 2 * self.config.downscale_factor

    @property
    def graph_epoch(self) -> int:
        return sum(a.graph_epoch for a in self.adapters)

    @torch.no_grad()
    def forward(self, xs: Sequence[torch.Tensor], adapter_weights: Optional[Sequence[float]] = None) -> List[torch.Tensor]:
        """One image per adapter -> the 4 combined features NHWC fp16; weights default to 1 / num_adapter each."""
        if len(xs) != self.num_adapter:
            raise IHError(f"MultiAdapter: {len(xs)} images for {self.num_adapter} adapters")
        w = [1.0 / self.num_adapter] * self.num_adapter if adapter_weights is None else [float(v) for v in adapter_weights]
        if len(w) != self.num_adapter:
            raise IHError(f"MultiAdapter: {len(w)} weights for {self.num_adapter} adapters")
        if any(tuple(x.shape) != tuple(xs[0].shape) for x in xs):
            raise IHError(f"MultiAdapter: the adapter images differ in shape {[tuple(x.shape) for x in xs]}")
        feats = [a(x) for a, x in zip(self.adapters, xs)]
        out = [torch.zeros_like(f) for f in feats[0]]
        dev = out[0].device
        scales = [torch.full((len(out),), wj, dtype=torch.float32, device=dev) for wj in w]   # fp32, as torch.tensor(w)
        ops.controlnet_add_residuals_multi(out, [[f.reshape(-1, f.shape[-1]) for f in fj] for fj in feats], scales,
                                           [0] * len(out))
        return out


@dataclass
class AdapterCall:
    """What DenoiseEngine.run(adapter=...) needs: the 4 adapter features NHWC fp16 [n, h_k, w_k, C_k], one row per image
    of the batch (a MultiAdapter's already combined), the scale the UNet multiplies them by (the single adapter's
    adapter_conditioning_scale; 1.0 for combined features) and keep[i] per schedule index (None: every step)."""
    features: Sequence[torch.Tensor]
    scale: float = 1.0
    keep: Optional[Sequence[float]] = None


def adapter_keep(num_steps: int, loop_steps: int, conditioning_factor: float) -> List[float]:
    """[3P] StableDiffusionXLAdapterPipeline: the adapter's features are added at step i iff
    i < int(num_inference_steps * adapter_conditioning_factor), num_inference_steps being the step count after the
    denoising_end cut (`loop_steps`).  One entry per index of the `num_steps`-step schedule."""
    active = int(loop_steps * conditioning_factor)
    return [1.0 if i < active else 0.0 for i in range(num_steps)]
