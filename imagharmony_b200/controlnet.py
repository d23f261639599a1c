"""SDXL ControlNetModel ([3P] diffusers 0.30.0, SURVEY appendix A.7) on the sm_90a kernel library.

The ControlNet is the UNet's encoder half with its own weights -- conv_in, the time and text_time embeddings, the down
blocks and the mid block, built from the UNet's block classes and run by the same code (unet.SDXLEncoderModel) --
plus a conditioning-image embedding added to conv_in's output and one 1x1 "zero conv" per residual.  State-dict keys
are diffusers' (`controlnet_cond_embedding.*`, `controlnet_down_blocks.{0..8}`, `controlnet_mid_block`).

`forward` returns the 10 zero-conv outputs UNSCALED with the device fp32 scale vector; the UNet multiplies and adds
them in one kernel (ops.controlnet_add_residuals), so a step graph captured once serves every conditioning scale.
The conditioning embedding is step-invariant: DenoiseEngine computes it once per call (`embed_condition`).
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
from .config import ControlNetConfig, config_from_diffusers
from .unet import DownBlock, MidBlock, SDXLEncoderModel, TimestepEmbedding


@dataclass
class ControlNetOutput:
    """residuals: the 10 zero-conv outputs [rows, C] fp16 (conv_in, every down-block resnet/attention and downsampler
    output, then the mid block), unscaled; scale: device fp32 [10], the factor of each."""
    residuals: List[torch.Tensor]
    scale: torch.Tensor


@dataclass
class ControlNetCall:
    """What DenoiseEngine.run(controlnet=...) needs: the model, the control image [n, 3, H, W] in [0, 1] (one per
    image of the batch, H x W = 8x the latents), the conditioning scale, guess mode, and keep[i] per schedule index
    (controlnet_keep; None runs the ControlNet at every step)."""
    model: "ControlNetModel"
    image: torch.Tensor
    conditioning_scale: float = 1.0
    guess_mode: bool = False
    keep: Optional[Sequence[float]] = None


def controlnet_scales(conditioning_scale: float, guess_mode: bool, n: int = 10) -> torch.Tensor:
    """[3P] diffusers ControlNetModel.forward's scaling of its n residuals as fp32 values (CPU): conditioning_scale for
    every one, or in guess mode torch.logspace(-1, 0, n)[k] * conditioning_scale (the last, the mid block's, at 1)."""
    if guess_mode:
        return torch.logspace(-1, 0, n) * float(conditioning_scale)
    return torch.full((n,), float(conditioning_scale), dtype=torch.float32)


def controlnet_keep(num_steps: int, start: float, end: float) -> List[float]:
    """[3P] StableDiffusionXLControlNetPipeline: keep[i] = 1 - (i/T < start or (i+1)/T > end) over the T steps of the
    schedule; the ControlNet runs at step i only where keep[i] = 1."""
    return [1.0 - float(i / num_steps < start or (i + 1) / num_steps > end) for i in range(num_steps)]


class ControlNetConditioningEmbedding(nn.Module):
    """conv_in (3 -> 16) + SiLU, then per consecutive width pair (c, c'): conv c -> c + SiLU, conv c -> c' stride 2 +
    SiLU; conv_out (-> 320) without activation.  All 3x3, pad 1.  The small-channel convs run on
    ops.conv3x3_small (bias + SiLU fused), conv_out on the implicit-GEMM conv."""

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int, block_out_channels):
        super().__init__()
        self.conv_in = nn.Conv2d(conditioning_channels, block_out_channels[0], 3, padding=1)
        blocks = []
        for c, c2 in zip(block_out_channels[:-1], block_out_channels[1:]):
            blocks.append(nn.Conv2d(c, c, 3, padding=1))
            blocks.append(nn.Conv2d(c, c2, 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        if block_out_channels[-1] % 64:
            raise IHError(f"ControlNet conditioning embedding: the last width ({block_out_channels[-1]}) must be a "
                          "multiple of 64 (conv_out runs on the implicit-GEMM conv)")
        self.conv_out = nn.Conv2d(block_out_channels[-1], conditioning_embedding_channels, 3, padding=1)
        self._w = None

    def finalize(self, bgr: bool) -> None:
        w_in = self.conv_in.weight.detach()
        if bgr:      # diffusers flips the image's channels first: conv(flip(x), W) = conv(x, W with flipped inputs)
            w_in = w_in.flip(1)
        self._w = [ops.pack_conv3x3_weight(w_in)] + [ops.pack_conv3x3_weight(b.weight.detach()) for b in self.blocks]
        self._w_out = ops.pack_conv3x3_weight(self.conv_out.weight.detach())

    def forward(self, image: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """image NCHW fp16 [B, 3, H, W] (values in [0, 1], the model's channel order not yet applied) -> NHWC fp16
        [B, H/8, W/8, 320]."""
        convs = [self.conv_in] + list(self.blocks)
        x = ops.conv3x3_small(image, self._w[0], self.conv_in.bias, silu=True, nchw=True)
        for conv, w in zip(convs[1:], self._w[1:]):
            x = ops.conv3x3_small(x, w, conv.bias, stride=conv.stride[0], silu=True)
        return ops.conv3x3(x, self._w_out, self.conv_out.bias, out=out)


class ControlNetModel(SDXLEncoderModel):
    """Native SDXL ControlNet. Build with `from_state_dict` / `from_pretrained`, or on the meta device +
    `load_state_dict(..., assign=True)` + `install_default_processors()` + `finalize()`."""

    def __init__(self, cfg: ControlNetConfig):
        super().__init__()
        if isinstance(cfg, (list, tuple)):
            raise IHError("ControlNetModel takes one config: wrap several ControlNets in MultiControlNetModel")
        if cfg.global_pool_conditions:
            raise IHError("ControlNet models with global_pool_conditions = true (shuffle-style, pooled residuals) are "
                          "not supported")
        if cfg.in_channels != 4:
            raise IHError(f"ControlNetModel: in_channels must be 4, got {cfg.in_channels}")
        if cfg.controlnet_conditioning_channel_order not in ("rgb", "bgr"):
            raise IHError(f"unknown controlnet_conditioning_channel_order "
                          f"{cfg.controlnet_conditioning_channel_order!r}")
        self.config = cfg
        boc = cfg.block_out_channels
        tl = cfg.transformer_layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], cfg.time_embed_dim)
        self.add_embedding = TimestepEmbedding(cfg.add_embed_in, cfg.time_embed_dim)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(boc[0], cfg.conditioning_channels,
                                                                         cfg.conditioning_embedding_out_channels)
        downs, res_ch = [], [boc[0]]
        ch = boc[0]
        for i, co in enumerate(boc):
            downs.append(DownBlock(cfg, ch, co, tl[i], add_down=i < len(boc) - 1))
            res_ch += [co] * (cfg.layers_per_block + (i < len(boc) - 1))
            ch = co
        self.down_blocks = nn.ModuleList(downs)
        self.controlnet_down_blocks = nn.ModuleList([nn.Conv2d(c, c, 1) for c in res_ch])
        self.controlnet_mid_block = nn.Conv2d(boc[-1], boc[-1], 1)
        self.mid_block = MidBlock(cfg, boc[-1], cfg.mid_depth)
        self._zc = None

    # ------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path: str, device="cuda", **kwargs) -> "ControlNetModel":
        """A diffusers ControlNet folder: config.json + diffusion_pytorch_model[.fp16].safetensors (keys strict)."""
        from safetensors.torch import load_file
        with open(os.path.join(path, "config.json")) as f:
            meta = json.load(f)
        if meta.get("global_pool_conditions", False):
            raise IHError("ControlNet models with global_pool_conditions = true are not supported")
        cfg = config_from_diffusers(meta, ControlNetConfig)
        for name in ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors"):
            f = os.path.join(path, name)
            if os.path.exists(f):
                return cls.from_state_dict(cfg, load_file(f), device=device)
        raise FileNotFoundError(f"no ControlNet weights (diffusion_pytorch_model[.fp16].safetensors) under {path}")

    def install_default_processors(self):
        """diffusers' default processors on a ControlNet: every token of encoder_hidden_states is a text token
        (CNAttnProcessor2_0 with num_tokens = 0); IPAdapter replaces them with num_tokens = its image tokens."""
        from ip_adapter.attention_processor import CNAttnProcessor2_0
        self.set_attn_processor(CNAttnProcessor2_0(num_tokens=0))

    def _finalize_ends(self):
        self._pack_conv_in()
        self.controlnet_cond_embedding.finalize(self.config.controlnet_conditioning_channel_order == "bgr")
        zcs = list(self.controlnet_down_blocks) + [self.controlnet_mid_block]
        self._zc = [(z.weight.detach().reshape(z.weight.shape[0], -1).contiguous(), z.bias.detach()) for z in zcs]

    # ------------------------------------------------------------------------------------------------------------
    def embed_condition(self, image: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The conditioning-image embedding: image NCHW fp16 [B, 3, H, W] in [0, 1] -> NHWC fp16 [B, H/8, W/8, 320]."""
        if self._zc is None:
            raise IHError("ControlNetModel.finalize() has not been called")
        return self.controlnet_cond_embedding(image, out=out)

    def forward(self, sample: torch.Tensor, timesteps: torch.Tensor, encoder_hidden_states: torch.Tensor,
                controlnet_cond: Optional[torch.Tensor] = None, conditioning_scale: float = 1.0,
                guess_mode: bool = False, text_embeds: Optional[torch.Tensor] = None,
                time_ids: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None,
                cond_embedding: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None) -> ControlNetOutput:
        """sample NCHW fp16 [B, 4, h, w]; timesteps / step as in UNet2DConditionModel.forward; controlnet_cond the
        control image NCHW fp16 [B, 3, 8h, 8w] in [0, 1], or `cond_embedding` its embedding NHWC [B, h, w, 320]
        (embed_condition).  The scale vector is controlnet_scales(conditioning_scale, guess_mode) on the device
        unless a device fp32 [10] `scale` is given."""
        B, _, h, w = sample.shape
        C0 = self.config.block_out_channels[0]
        if cond_embedding is None:
            if controlnet_cond is None:
                raise IHError("ControlNetModel.forward needs controlnet_cond (the control image) or cond_embedding")
            if tuple(controlnet_cond.shape) != (B, self.config.conditioning_channels, 8 * h, 8 * w):
                raise IHError(f"controlnet_cond: expected {(B, self.config.conditioning_channels, 8 * h, 8 * w)}, got "
                              f"{tuple(controlnet_cond.shape)}")
            cond_embedding = self.embed_condition(controlnet_cond)
        if tuple(cond_embedding.shape) != (B, h, w, C0):
            raise IHError(f"cond_embedding: expected {(B, h, w, C0)}, got {tuple(cond_embedding.shape)}")
        if scale is None:
            scale = controlnet_scales(conditioning_scale, guess_mode, len(self._zc)).to(sample.device)
        self._ensure_conditioning(encoder_hidden_states, text_embeds, time_ids, B)
        temb_all = self.time_embeddings(timesteps, step, B)
        a = ops.im2col3x3_nchw(sample, self._w_in.shape[1])
        x = ops.linear(a, self._w_in, self.conv_in.bias, residual=cond_embedding.reshape(B * h * w, C0))   # DESIGN §4
        x = x.reshape(B, h, w, C0)
        skips = [x]
        for blk in self.down_blocks:
            x = blk(x, temb_all, encoder_hidden_states, skips)
        x = self.mid_block(x, temb_all, encoder_hidden_states)
        res = [ops.linear(t.reshape(-1, t.shape[-1]), wz, bz) for t, (wz, bz) in zip(skips + [x], self._zc)]
        return ControlNetOutput(res, scale)


class MultiControlNetModel(nn.Module):
    """[3P] diffusers MultiControlNetModel: several ControlNets (`.nets`) whose scaled residuals are summed, in fp16 and
    in net order, before the UNet adds them.  DenoiseEngine does not call `forward`: it runs the nets one by one and
    sums and injects their residuals in one kernel (ops.controlnet_add_residuals_multi), with the same rounding."""

    def __init__(self, nets):
        super().__init__()
        nets = list(nets)
        if not nets:
            raise IHError("Multi-ControlNet: the list of ControlNets is empty")
        if len(nets) > IH_CN_MAX_NETS:
            raise IHError(f"Multi-ControlNet: {len(nets)} ControlNets, at most {IH_CN_MAX_NETS} are supported")
        for i, net in enumerate(nets):
            if not isinstance(net, ControlNetModel):
                raise IHError(f"Multi-ControlNet: entry {i} is {type(net).__name__}, not a ControlNetModel")
        boc = nets[0].config.block_out_channels
        for i, net in enumerate(nets):
            if net.config.block_out_channels != boc:
                raise IHError(f"Multi-ControlNet: net {i} has block_out_channels {net.config.block_out_channels}, "
                              f"net 0 has {boc}")
        self.nets = nn.ModuleList(nets)

    def forward(self, sample: torch.Tensor, timesteps: torch.Tensor, encoder_hidden_states: torch.Tensor,
                controlnet_cond: Sequence[torch.Tensor], conditioning_scale: Sequence[float], guess_mode: bool = False,
                text_embeds: Optional[torch.Tensor] = None, time_ids: Optional[torch.Tensor] = None,
                step: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        """The eager sum: one control image and conditioning scale per net -> the 10 summed SCALED residuals [rows, C]
        (residual_k * scale_k of each net in its dtype, then added in net order)."""
        if len(controlnet_cond) != len(self.nets) or len(conditioning_scale) != len(self.nets):
            raise IHError(f"Multi-ControlNet: {len(controlnet_cond)} images and {len(conditioning_scale)} scales for "
                          f"{len(self.nets)} nets")
        total = None
        for net, image, cs in zip(self.nets, controlnet_cond, conditioning_scale):
            out = net(sample, timesteps, encoder_hidden_states, controlnet_cond=image, conditioning_scale=cs,
                      guess_mode=guess_mode, text_embeds=text_embeds, time_ids=time_ids, step=step)
            scaled = [(r.float() * s).to(r.dtype) for r, s in zip(out.residuals, out.scale)]
            total = scaled if total is None else [a + b for a, b in zip(total, scaled)]
        return total
