"""Native SDXL tiny autoencoder decoder (TAESD-XL): `pipe.vae = AutoencoderTiny.from_pretrained(dir)`.

Module tree and state-dict keys are those of [3P] diffusers `AutoencoderTiny` / `DecoderTiny` (`decoder.layers.*`;
the encoder keys of a full checkpoint are ignored), restated from the published structure, parity unpinned:

    x = tanh(x / 3) * 3
    Conv(L, C), ReLU
    per stage i: num_decoder_blocks[i] x Block; except after the last stage: nearest 2x Upsample, Conv(C, C, bias=False)
    Conv(C, out_channels)
    x * 2 - 1

Block(x) = relu(conv3(relu(conv2(relu(conv1(x))))) + x).  A 64-channel, GroupNorm-free decoder: about 19x fewer FLOPs
than the KL decoder at the same image size (tools/bench_taesd.py counts both).

Every conv runs on the implicit-GEMM kernel of this package, the ReLUs in its epilogue (IH_EPI_RELU, applied after the
residual, so a whole Block is three launches):

* the clamp is the same fp16 torch expression as diffusers' on the tiny [B, L, h, w] latent (elementwise glue);
* conv_in (3x3, L -> C): `ih_im2col3x3_nchw_f16` [B*h*w, 9 L -> 64] + one GEMM with the ReLU epilogue;
* Block: three 3x3 convs with the ReLU epilogue, the third with the block input as its residual;
* Upsample: `ih_upsample2x_f16`, then the bias-free 3x3 conv;
* conv_out: Cout padded to 16, `* 2 - 1` folded into the epilogue as alpha = 2 and bias 2 b - 1, then a gather to NCHW.
  It rounds once, fp16(2 acc + fp16(2 b - 1)), where diffusers rounds the conv output and the subtraction,
  fp16(2 fp16(acc + b) - 1); the two differ by about one fp16 ulp of the output.

Tiling is not restated: with `use_tiling` (pipe.enable_vae_tiling()) `decode` raises, so an image diffusers would decode
in blended tiles is never silently decoded whole.  The tiny encoder is not built: image-to-image and inpainting refuse
to encode a pixel image while `pipe.vae` is a tiny autoencoder.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List

import torch
import torch.nn as nn

from . import ops
from ._lib import IHError
from .config import TAESDXL, TinyVAEConfig

_KPAD = 64          # conv_in's im2col row width: 9 L <= 64
_OUT_PAD = 16       # conv_out's Cout padded for the conv kernel's tiles


class TinyBlock(nn.Module):
    """[3P] AutoencoderTinyBlock with in_channels == out_channels (identity skip, ReLU fuse)."""

    def __init__(self, ch: int):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(ch, ch, 3, padding=1), nn.ReLU(), nn.Conv2d(ch, ch, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(ch, ch, 3, padding=1))
        self.skip = nn.Identity()
        self.fuse = nn.ReLU()
        self._w = self._b = None

    def finalize(self):
        convs = (self.conv[0], self.conv[2], self.conv[4])
        self._w = [ops.pack_conv3x3_weight(c.weight.detach()) for c in convs]
        self._b = [c.bias.detach() for c in convs]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = ops.conv3x3(x, self._w[0], self._b[0], relu=True)
        h = ops.conv3x3(h, self._w[1], self._b[1], relu=True)
        return ops.conv3x3(h, self._w[2], self._b[2], residual=x, relu=True)


class DecoderTiny(nn.Module):
    def __init__(self, cfg: TinyVAEConfig):
        super().__init__()
        ch = cfg.decoder_block_out_channels
        layers: List[nn.Module] = [nn.Conv2d(cfg.latent_channels, ch[0], 3, padding=1), nn.ReLU()]
        for i, n in enumerate(cfg.num_decoder_blocks):
            last = i == len(cfg.num_decoder_blocks) - 1
            layers += [TinyBlock(ch[i]) for _ in range(n)]
            if not last:
                layers.append(nn.Upsample(scale_factor=2, mode="nearest"))
            layers.append(nn.Conv2d(ch[i], cfg.out_channels if last else ch[i], 3, padding=1, bias=last))
        self.layers = nn.Sequential(*layers)


def check_config(meta: dict) -> TinyVAEConfig:
    """A diffusers AutoencoderTiny config.json -> TinyVAEConfig; IHError for every value the native decoder does not
    implement."""
    for key, want in (("act_fn", "relu"), ("upsample_fn", "nearest"), ("upsampling_scaling_factor", 2)):
        if key in meta and meta[key] != want:
            raise IHError(f"AutoencoderTiny: {key} = {meta[key]!r} is not implemented (only {want!r})")
    d = TAESDXL
    ch = tuple(int(c) for c in meta.get("decoder_block_out_channels", d.decoder_block_out_channels))
    blocks = tuple(int(n) for n in meta.get("num_decoder_blocks", d.num_decoder_blocks))
    if len(ch) != len(blocks) or not ch:
        raise IHError(f"AutoencoderTiny: decoder_block_out_channels {ch} and num_decoder_blocks {blocks} differ in length")
    if any(c % 64 or c != ch[0] for c in ch):
        raise IHError(f"AutoencoderTiny: decoder_block_out_channels {ch} must be one width, a multiple of 64 (the "
                      "implicit-GEMM conv needs Cin % 64 == 0; diffusers' DecoderTiny chains equal widths)")
    cfg = TinyVAEConfig(latent_channels=int(meta.get("latent_channels", d.latent_channels)),
                        out_channels=int(meta.get("out_channels", d.out_channels)), decoder_block_out_channels=ch,
                        num_decoder_blocks=blocks, scaling_factor=float(meta.get("scaling_factor", d.scaling_factor)))
    if not 1 <= cfg.latent_channels <= _KPAD // 9 or not 1 <= cfg.out_channels <= _OUT_PAD:
        raise IHError(f"AutoencoderTiny: latent_channels {cfg.latent_channels} (at most {_KPAD // 9}) or out_channels "
                      f"{cfg.out_channels} (at most {_OUT_PAD}) not implemented")
    return cfg


class AutoencoderTinyDecoder(nn.Module):
    """`decode(latents)` = diffusers `AutoencoderTiny.decode(latents / scaling_factor).sample` (the division is folded
    in), so the pipelines' `_output` and `postprocess` treat it like `AutoencoderKLDecoder`."""

    def __init__(self, cfg: TinyVAEConfig = TAESDXL):
        super().__init__()
        self.config = cfg
        self.decoder = DecoderTiny(cfg)
        self.use_tiling = False             # pipe.enable_vae_tiling(): decode then refuses (module docstring)
        self._w_in = None

    # ---- construction ------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=torch.float16, device="cuda") -> "AutoencoderTinyDecoder":
        """A diffusers AutoencoderTiny folder (e.g. madebyollin/taesdxl): config.json +
        diffusion_pytorch_model[.fp16].safetensors."""
        if torch_dtype != torch.float16:
            raise IHError(f"AutoencoderTiny runs in fp16 (torch_dtype={torch_dtype} requested)")
        from safetensors.torch import load_file
        with open(os.path.join(path, "config.json")) as f:
            cfg = check_config(json.load(f))
        for name in ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors"):
            f = os.path.join(path, name)
            if os.path.exists(f):
                return cls.from_state_dict(cfg, load_file(f), device=device)
        raise FileNotFoundError(f"no AutoencoderTiny weights (diffusion_pytorch_model[.fp16].safetensors) under {path}")

    @classmethod
    def from_state_dict(cls, cfg: TinyVAEConfig, sd: Dict[str, torch.Tensor], device="cuda") -> "AutoencoderTinyDecoder":
        """`sd` may hold the encoder too: only `decoder.*` is read, and it must be exactly the decoder `cfg` builds."""
        with torch.device("meta"):
            m = cls(cfg)
        own = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        have = {k: tuple(v.shape) for k, v in sd.items() if k.startswith("decoder.")}
        missing, extra = sorted(set(own) - set(have)), sorted(set(have) - set(own))
        shapes = sorted(k for k in set(own) & set(have) if own[k] != have[k])
        if missing or extra or shapes:
            raise IHError(f"AutoencoderTiny: the checkpoint's decoder does not match num_decoder_blocks "
                          f"{cfg.num_decoder_blocks} / decoder_block_out_channels {cfg.decoder_block_out_channels}: "
                          f"missing {missing[:3]}, unexpected {extra[:3]}, other shapes {shapes[:3]}")
        m = m.to_empty(device=device)
        m.load_state_dict({k: sd[k].to(device=device, dtype=torch.float16) for k in own})
        m = m.half().eval()
        m.finalize()
        return m

    def finalize(self) -> None:
        layers = self.decoder.layers
        for mod in layers:
            if isinstance(mod, TinyBlock):
                mod.finalize()
        ci, co = layers[0], layers[-1]
        C, L = ci.weight.shape[0], ci.weight.shape[1]
        w = torch.zeros((C, _KPAD), dtype=ci.weight.dtype, device=ci.weight.device)
        w[:, :L * 9] = ci.weight.detach().reshape(C, L * 9)                          # k = ci*9 + ky*3 + kx
        self._w_in, self._b_in = w.contiguous(), ci.bias.detach()
        self._w_up = [ops.pack_conv3x3_weight(m.weight.detach()) for m in layers[1:-1] if isinstance(m, nn.Conv2d)]
        wo = torch.zeros((_OUT_PAD,) + tuple(co.weight.shape[1:]), dtype=co.weight.dtype, device=co.weight.device)
        wo[:co.weight.shape[0]] = co.weight.detach()
        self._w_out = ops.pack_conv3x3_weight(wo)
        bo = torch.zeros((_OUT_PAD,), dtype=torch.float32, device=co.weight.device)
        bo[:co.weight.shape[0]] = co.bias.detach().float() * 2 - 1                   # x * 2 - 1 (alpha = 2 in decode)
        self._b_out = bo.to(co.weight.dtype)

    # ---- forward -----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def decode(self, latents: torch.Tensor) -> torch.Tensor:
        """latents [B, L, h, w] fp16 straight from the denoise loop -> image [B, 3, 8h, 8w] fp16 in [-1, 1] (nominally)."""
        if self._w_in is None:
            raise IHError("AutoencoderTinyDecoder.finalize() has not run (use from_pretrained / from_state_dict)")
        if self.use_tiling:
            raise IHError("AutoencoderTiny: tiled decoding (enable_vae_tiling) is not implemented; diffusers blends "
                          "tiles that an untiled decode would not reproduce")
        cfg = self.config
        if latents.dim() != 4 or latents.shape[1] != cfg.latent_channels:
            raise IHError(f"AutoencoderTiny.decode: expected [B, {cfg.latent_channels}, h, w], got {tuple(latents.shape)}")
        B, _, h, w = latents.shape
        x = latents.to(self._w_in.dtype)
        if cfg.scaling_factor != 1.0:
            x = x / cfg.scaling_factor
        x = (torch.tanh(x / 3) * 3).contiguous()                                     # DecoderTiny's clamp
        a = ops.im2col3x3_nchw(x, _KPAD)
        x = ops.linear(a, self._w_in, self._b_in, relu=True).reshape(B, h, w, -1)    # conv_in + ReLU
        ups = iter(self._w_up)
        for mod in self.decoder.layers[2:-1]:
            if isinstance(mod, TinyBlock):
                x = mod(x)
            elif isinstance(mod, nn.Upsample):
                x = ops.conv3x3(ops.upsample2x(x), next(ups))                        # Upsample + Conv(bias=False)
        x = ops.conv3x3(x, self._w_out, self._b_out, alpha=2.0)                      # conv_out, * 2 - 1
        return ops.nhwc_to_nchw(x, cfg.out_channels)


AutoencoderTiny = AutoencoderTinyDecoder    # diffusers' class name: `pipe.vae = AutoencoderTiny.from_pretrained(dir)`

