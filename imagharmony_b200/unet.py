"""SDXL UNet2DConditionModel running on the sm_90a kernel library.

Same module tree / state-dict keys / `attn_processors` + `set_attn_processor` surface as the diffusers model the
reference drives (ip_adapter.py:102,125; custom_pipelines.py:338-345), but the forward pass is a sequence of C-ABI
kernel launches on NHWC fp16 activations:

    conv_in -> [ResBlock: GN+SiLU -> conv3x3(+temb) -> GN+SiLU -> conv3x3(+shortcut/residual)]
            -> [Transformer2D: GN -> proj_in -> N x (LN -> fused-QKV GEMM -> attention -> out GEMM(+res);
                                                    LN -> q GEMM -> decoupled IP cross attention -> out GEMM(+res);
                                                    LN -> GEGLU GEMM -> FF-out GEMM(+res)) -> proj_out(+res)]
            -> ... -> GN+SiLU -> conv_out

nn.Linear / nn.Conv2d / nn.GroupNorm / nn.LayerNorm instances are used purely as parameter containers (their own
forward is never called); kernel-layout copies (tap-major conv weights, fused QKV / KV matrices, the concatenated
time_emb_proj matrix) are derived once in `finalize()`.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import ops
from ._lib import IHError
from .config import UNetConfig


def adapter_targets(cfg: UNetConfig, h: int, w: int) -> List[tuple]:
    """(h, w, C) of the points where [3P] diffusers' UNet2DConditionModel adds down_intrablock_additional_residuals
    (T2I-Adapter features), in the order it takes them: one per down block -- after the block (after its downsampler)
    for a block without cross-attention, after its last resnet / attention pair for one with -- then, last, the mid
    block's output, which takes a leftover feature only if the shapes are equal."""
    out = []
    for i, co in enumerate(cfg.block_out_channels):
        down = i < len(cfg.block_out_channels) - 1 and cfg.transformer_layers_per_block[i] == 0
        s = 2 ** (i + down)
        out.append((h // s, w // s, co))
    s = 2 ** (len(cfg.block_out_channels) - 1)
    out.append((h // s, w // s, cfg.block_out_channels[-1]))
    return out


def require_adapter_shapes(cfg: UNetConfig, h: int, w: int, shapes) -> None:
    """IHError unless T2I-Adapter features of (h, w, C) `shapes` each land on an injection point of this UNet at an
    h x w latent (adapter_targets), every one of them used, as diffusers would add them."""
    targets = adapter_targets(cfg, h, w)
    shapes = [tuple(int(v) for v in s) for s in shapes]
    n_down = len(targets) - 1
    ok = len(shapes) <= n_down + 1 and all(s == t for s, t in zip(shapes, targets[:n_down]))
    if ok and len(shapes) == n_down + 1:
        ok = shapes[-1] == targets[-1]
    if not ok:
        raise IHError(f"T2I-Adapter features (h, w, C) {shapes} do not match this UNet's injection points {targets} at a "
                      f"{h}x{w} latent (its down blocks, then the mid block): the adapter's channels must equal the "
                      f"UNet's block_out_channels {list(cfg.block_out_channels)} plus the mid block's")


def require_latent_size(cfg: UNetConfig, h: int, w: int) -> None:
    """IHError unless an h x w latent fits the UNet: each of its len(block_out_channels) - 1 stride-2 downsamplers
    halves the sides exactly, and every up-block upsamples to twice its input, so both sides must be divisible by
    2 ** (len(block_out_channels) - 1) latents (4 for SDXL: images whose sides are multiples of 32 pixels)."""
    m = 2 ** (len(cfg.block_out_channels) - 1)
    if h % m or w % m:
        raise IHError(f"latent size {h}x{w} ({8 * h}x{8 * w} pixels) is not supported: the UNet needs latent sides "
                      f"divisible by {m}, i.e. image heights and widths that are multiples of {8 * m} pixels")


class Attention(nn.Module):
    """Parameter shell with the attributes the reference processors read (attention_processor.py:374-463)."""

    def __init__(self, query_dim: int, heads: int, cross_attention_dim: Optional[int] = None):
        super().__init__()
        kv_dim = cross_attention_dim or query_dim
        self.heads = heads
        self.is_cross = cross_attention_dim is not None
        self.to_q = nn.Linear(query_dim, query_dim, bias=False)
        self.to_k = nn.Linear(kv_dim, query_dim, bias=False)
        self.to_v = nn.Linear(kv_dim, query_dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(query_dim, query_dim), nn.Dropout(0.0)])
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = False
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.processor = None
        self._w_qkv = None
        self._w_kv = None
        self._ln = None      # (gamma-scaled centred weight, constant vector) of the projection that consumes a folded LayerNorm
        self._next_w = None  # weight of the GEMM that runs after this attention's out projection (L2 prefetch hint)

    def fold_ln(self, norm: nn.LayerNorm) -> None:
        """Fold the block's LayerNorm into the first projection of this attention (q|k|v for attn1, q for attn2)."""
        w = self.to_q.weight.detach() if self.is_cross else self.fused_qkv_weight()
        self._ln = ops.fold_layernorm(w, None, norm.weight.detach(), norm.bias.detach())

    def fused_qkv_weight(self) -> torch.Tensor:
        if self._w_qkv is None:
            self._w_qkv = torch.cat([self.to_q.weight.detach(), self.to_k.weight.detach(),
                                     self.to_v.weight.detach()], dim=0).contiguous()
        return self._w_qkv

    def fused_kv_weight(self) -> torch.Tensor:
        if self._w_kv is None:
            self._w_kv = torch.cat([self.to_k.weight.detach(), self.to_v.weight.detach()], dim=0).contiguous()
        return self._w_kv

    def drop_fused(self):
        self._w_qkv = None
        self._w_kv = None
        self._ln = None
        self._next_w = None

    def first_weight(self) -> torch.Tensor:
        """The weight the first GEMM of this attention streams (folded-LayerNorm form when it exists)."""
        if self._ln is not None:
            return self._ln[0]
        return self.to_q.weight.detach() if self.is_cross else self.fused_qkv_weight()   # detach: never register as a parameter

    def forward(self, hidden_states, encoder_hidden_states=None, **fused):
        """`fused` carries the native-processor extensions (residual=, ln_stats=, ln_eps=, stats_out=)."""
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states, attention_mask=None,
                              **fused)


class ResnetBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, temb_dim: int, groups: int):
        super().__init__()
        self.cin, self.cout, self.groups = cin, cout, groups
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-5)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_dim, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-5)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self._w1 = self._w2 = self._wsc = None
        self.temb_offset = 0   # column offset of this block inside the concatenated time_emb_proj output

    def finalize(self):
        self._w1 = ops.pack_conv3x3_weight(self.conv1.weight.detach())
        self._w2 = ops.pack_conv3x3_weight(self.conv2.weight.detach())
        if self.conv_shortcut is not None:
            self._wsc = self.conv_shortcut.weight.detach().reshape(self.cout, self.cin).contiguous()
            # conv2 with the 1x1 shortcut (and the skip concat of the up-blocks) as extra K blocks of the same launch
            self._w2sc = torch.cat([self._w2, self._wsc], dim=1).contiguous()
            self._b2sc = (self.conv2.bias.detach().float() + self.conv_shortcut.bias.detach().float()).to(self._w2.dtype)

    def forward(self, x: torch.Tensor, temb_all: torch.Tensor, skip: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x NHWC [B,H,W,C0] (+ skip [B,H,W,C1] concatenated on channels); temb_all [B, sum(Cout)]."""
        B, H, W, _ = x.shape
        h = ops.groupnorm(x, self.norm1.weight, self.norm1.bias, x1=skip, groups=self.groups, eps=1e-5, silu=True)
        temb = temb_all[:, self.temb_offset:self.temb_offset + self.cout]
        ops.prefetch_next(self._w2)
        h = ops.conv3x3(h, self._w1, self.conv1.bias, rowbias=temb)
        h = ops.groupnorm(h, self.norm2.weight, self.norm2.bias, groups=self.groups, eps=1e-5, silu=True)
        if self.conv_shortcut is not None:
            c0, c1 = x.shape[-1], (0 if skip is None else skip.shape[-1])
            if c0 % 64 == 0 and c1 % 64 == 0:      # every SDXL ResBlock: shortcut + concat fused into conv2
                return ops.conv3x3(h, self._w2sc, self._b2sc, shortcut=(x, skip))
            xin = x if skip is None else ops.concat_channels(x, skip)
            sc = ops.linear(xin.reshape(B * H * W, self.cin), self._wsc, self.conv_shortcut.bias)
            sc = sc.reshape(B, H, W, self.cout)
        else:
            if skip is not None:
                raise IHError("ResnetBlock2D: concatenated input needs a conv_shortcut")
            sc = x
        return ops.conv3x3(h, self._w2, self.conv2.bias, residual=sc)


class GEGLU(nn.Module):
    def __init__(self, dim: int, inner: int):
        super().__init__()
        self.proj = nn.Linear(dim, inner * 2)


class FeedForward(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim: int, heads: int, cross_dim: int):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        self.attn1 = Attention(dim, heads)
        self.norm2 = nn.LayerNorm(dim, eps=1e-5)
        self.attn2 = Attention(dim, heads, cross_dim)
        self.norm3 = nn.LayerNorm(dim, eps=1e-5)
        self.ff = FeedForward(dim)
        self._ln_ff = None
        self._next_w = None       # weight of the GEMM after this block's FF-out (next block's q|k|v, or proj_out)

    def finalize(self):
        self.attn1.fold_ln(self.norm1)
        self.attn2.fold_ln(self.norm2)
        self._ln_ff = ops.fold_layernorm(self.ff.net[0].proj.weight.detach(), self.ff.net[0].proj.bias.detach(),
                                         self.norm3.weight.detach(), self.norm3.bias.detach())
        # L2 prefetch chain inside the block: attn1.out -> attn2 q weight, attn2.out -> GEGLU weight
        self.attn1._next_w = self.attn2.first_weight()
        self.attn2._next_w = self._ln_ff[0]

    def _attend(self, attn, norm, h, ehs, h_stats, want_stats):
        """h + attn(norm(h)) with the LayerNorm folded into the attention's first GEMM when row statistics of `h`
        are available (written by the GEMM that produced `h`).  Returns (new h, its row statistics or None)."""
        B, N, C = h.shape
        proc = attn.processor
        if not getattr(proc, "supports_fused", False):
            # foreign processor: plain diffusers protocol (normalised input, no fused residual)
            n = ops.layernorm(h, norm.weight, norm.bias, norm.eps)
            out = proc(attn, n, encoder_hidden_states=ehs, attention_mask=None)
            return ops.add_bcast(h, out.contiguous()), None
        st = torch.empty((C // 64, B * N, 2), dtype=torch.float32, device=h.device) if want_stats else None
        if h_stats is not None and attn._ln is not None:
            return attn(h, ehs, residual=h, ln_stats=h_stats, ln_eps=norm.eps, stats_out=st), st
        n = ops.layernorm(h, norm.weight, norm.bias, norm.eps)
        return attn(n, ehs, residual=h, stats_out=st), st

    def forward(self, h: torch.Tensor, ehs: torch.Tensor, h_stats: Optional[torch.Tensor] = None, want_stats=True):
        """h [B, N, C] tokens; h_stats: per-row (sum, sumsq) slabs of h written by the producing GEMM (or None)."""
        B, N, C = h.shape
        fold = C % 64 == 0
        h, st = self._attend(self.attn1, self.norm1, h, None, h_stats if fold else None, fold)
        h, st = self._attend(self.attn2, self.norm2, h, ehs, st, fold)
        h2d = h.reshape(B * N, C)
        ops.prefetch_next(self.ff.net[2].weight)
        if st is not None and self._ln_ff is not None:
            w_c, c = self._ln_ff
            g = ops.linear(h2d, w_c, c, geglu=True, ln=(st, self.norm3.eps))
        else:
            n = ops.layernorm(h, self.norm3.weight, self.norm3.bias, self.norm3.eps)
            g = ops.linear(n.reshape(B * N, C), self.ff.net[0].proj.weight, self.ff.net[0].proj.bias, geglu=True)
        st_out = torch.empty((C // 64, B * N, 2), dtype=torch.float32, device=h.device) if (fold and want_stats) else None
        ops.prefetch_next(self._next_w)
        h2 = ops.linear(g, self.ff.net[2].weight, self.ff.net[2].bias, residual=h2d, stats_out=st_out)
        return h2.reshape(B, N, C), st_out


class Transformer2DModel(nn.Module):
    def __init__(self, dim: int, heads: int, depth: int, cross_dim: int, groups: int):
        super().__init__()
        self.groups = groups
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        self.proj_in = nn.Linear(dim, dim)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, heads, cross_dim) for _ in range(depth)])
        self.proj_out = nn.Linear(dim, dim)

    def link_prefetch(self):
        """FF-out of block i hints block i + 1's first weight (the last block hints proj_out); proj_in hints block 0."""
        blocks = list(self.transformer_blocks)
        for i, blk in enumerate(blocks):
            blk._next_w = blocks[i + 1].attn1.first_weight() if i + 1 < len(blocks) else self.proj_out.weight.detach()

    def forward(self, x: torch.Tensor, ehs: torch.Tensor) -> torch.Tensor:
        B, H, W, C = x.shape
        h = ops.groupnorm(x, self.norm.weight, self.norm.bias, groups=self.groups, eps=1e-6, silu=False)
        st = torch.empty((C // 64, B * H * W, 2), dtype=torch.float32, device=x.device) if C % 64 == 0 else None
        ops.prefetch_next(self.transformer_blocks[0].attn1.first_weight())
        h = ops.linear(h.reshape(B * H * W, C), self.proj_in.weight, self.proj_in.bias, stats_out=st)
        h = h.reshape(B, H * W, C)
        nblk = len(self.transformer_blocks)
        for i, blk in enumerate(self.transformer_blocks):
            h, st = blk(h, ehs, st, want_stats=i + 1 < nblk)
        out = ops.linear(h.reshape(B * H * W, C), self.proj_out.weight, self.proj_out.bias,
                         residual=x.reshape(B * H * W, C))
        return out.reshape(B, H, W, C)


class Resample(nn.Module):
    def __init__(self, ch: int, up: bool):
        super().__init__()
        self.up = up
        self.conv = nn.Conv2d(ch, ch, 3, stride=1 if up else 2, padding=1)
        self._w = None

    def finalize(self):
        self._w = ops.pack_conv3x3_weight(self.conv.weight.detach())

    def forward(self, x):
        if self.up:
            return ops.conv3x3(ops.upsample2x(x), self._w, self.conv.bias)
        return ops.conv3x3(x, self._w, self.conv.bias, stride=2)


class DownBlock(nn.Module):
    def __init__(self, cfg: UNetConfig, cin: int, cout: int, depth: int, add_down: bool):
        super().__init__()
        temb = cfg.time_embed_dim
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, temb, cfg.norm_num_groups)
                                      for j in range(cfg.layers_per_block)])
        self.has_attn = depth > 0
        if self.has_attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, cfg.heads(cout), depth, cfg.cross_attention_dim,
                                                                cfg.norm_num_groups)
                                             for _ in range(cfg.layers_per_block)])
        self.has_down = add_down
        if add_down:
            self.downsamplers = nn.ModuleList([Resample(cout, up=False)])

    def forward(self, x, temb_all, ehs, skips: List[torch.Tensor], inject=None):
        """`inject(x)`: an in-place addition to the output of the last resnet / attention pair, before it is appended
        to the skips and downsampled (diffusers' additional_residuals of CrossAttnDownBlock2D)."""
        for j, res in enumerate(self.resnets):
            x = res(x, temb_all)
            if self.has_attn:
                x = self.attentions[j](x, ehs)
            if inject is not None and j == len(self.resnets) - 1:
                inject(x)
            skips.append(x)
        if self.has_down:
            x = self.downsamplers[0](x)
            skips.append(x)
        return x


class MidBlock(nn.Module):
    def __init__(self, cfg: UNetConfig, ch: int, depth: int):
        super().__init__()
        temb = cfg.time_embed_dim
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb, cfg.norm_num_groups) for _ in range(2)])
        self.attentions = nn.ModuleList([Transformer2DModel(ch, cfg.heads(ch), depth, cfg.cross_attention_dim,
                                                            cfg.norm_num_groups)])

    def forward(self, x, temb_all, ehs):
        x = self.resnets[0](x, temb_all)
        x = self.attentions[0](x, ehs)
        return self.resnets[1](x, temb_all)


class UpBlock(nn.Module):
    def __init__(self, cfg: UNetConfig, prev_out: int, skip_ch: int, cout: int, depth: int, add_up: bool):
        super().__init__()
        temb = cfg.time_embed_dim
        n = cfg.layers_per_block + 1
        res = []
        for j in range(n):
            res_skip = skip_ch if j == n - 1 else cout
            res_in = prev_out if j == 0 else cout
            res.append(ResnetBlock2D(res_in + res_skip, cout, temb, cfg.norm_num_groups))
        self.resnets = nn.ModuleList(res)
        self.has_attn = depth > 0
        if self.has_attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, cfg.heads(cout), depth, cfg.cross_attention_dim,
                                                                cfg.norm_num_groups) for _ in range(n)])
        self.has_up = add_up
        if add_up:
            self.upsamplers = nn.ModuleList([Resample(cout, up=True)])

    def forward(self, x, temb_all, ehs, skips: List[torch.Tensor]):
        for j, res in enumerate(self.resnets):
            x = res(x, temb_all, skip=skips.pop())     # GN / shortcut read the two tensors; no standalone concat
            if self.has_attn:
                x = self.attentions[j](x, ehs)
        if self.has_up:
            x = self.upsamplers[0](x)
        return x


class TimestepEmbedding(nn.Module):
    def __init__(self, in_dim: int, dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_dim, dim)
        self.linear_2 = nn.Linear(dim, dim)


class SDXLEncoderModel(nn.Module):
    """What the UNet and the ControlNet share: processor plumbing (`attn_processors` / `set_attn_processor`), the
    kernel-layout weights of the blocks (`finalize`), the step-invariant conditioning (`prepare_conditioning`: the
    cross-attention K/V and the text_time embedding) and the per-step time embeddings.  Subclasses own `conv_in`,
    `time_embedding`, `add_embedding`, the blocks, and `_finalize_ends()` for the weights outside the blocks."""

    def __init__(self):
        super().__init__()
        self._w_temb = None
        self._b_temb = None
        self._aug = None          # (key, aug_emb [B, time_embed_dim]) of the last prepare_conditioning()
        self._aug_bufs = {}       # B -> buffer; kept for the life of the model: captured CUDA graphs point at them
        self._text_only = None
        self.graph_epoch = 0      # bumped when weights / processors change: graphs captured earlier are stale

    # ------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_state_dict(cls, cfg, state_dict: Dict[str, torch.Tensor], device="cuda"):
        with torch.device("meta"):
            m = cls(cfg)
        sd = {k: v.to(device=device, dtype=torch.float16) for k, v in state_dict.items()}
        m.load_state_dict(sd, assign=True)
        m.requires_grad_(False)
        m.install_default_processors()
        m.finalize()
        return m

    def _attn_modules(self):
        for name, m in self.named_modules():
            if isinstance(m, Attention):
                yield name, m

    @property
    def attn_processors(self) -> Dict[str, object]:
        return {f"{name}.processor": m.processor for name, m in self._attn_modules()}

    def set_attn_processor(self, procs) -> None:
        for name, m in self._attn_modules():
            m.processor = procs[f"{name}.processor"] if isinstance(procs, dict) else procs
        self.graph_epoch += 1

    def finalize(self):
        """Derive kernel-layout weights. Call after (re)loading parameters."""
        offs = 0
        ws, bs = [], []
        for m in self.modules():
            if isinstance(m, (ResnetBlock2D, Resample)):
                m.finalize()
            if isinstance(m, BasicTransformerBlock):
                m._ln_ff = None
            if isinstance(m, ResnetBlock2D):
                m.temb_offset = offs
                offs += m.cout
                ws.append(m.time_emb_proj.weight.detach())
                bs.append(m.time_emb_proj.bias.detach())
            if isinstance(m, Attention):
                m.drop_fused()
                (m.fused_kv_weight() if m.is_cross else m.fused_qkv_weight())
        for m in self.modules():      # after the fused q|k|v weights exist: fold the LayerNorms into their consumers
            if isinstance(m, BasicTransformerBlock):
                m.finalize()
        for m in self.modules():
            if isinstance(m, Transformer2DModel):
                m.link_prefetch()
        self._w_temb = torch.cat(ws, 0).contiguous()
        self._b_temb = torch.cat(bs, 0).contiguous()
        self._finalize_ends()
        self._aug = None
        for p in self.attn_processors.values():
            if hasattr(p, "invalidate"):
                p.invalidate()
        self.graph_epoch += 1

    def _finalize_ends(self):
        raise NotImplementedError

    def _pack_conv_in(self):
        """conv_in runs on the tensor-core GEMM over ops.im2col3x3_nchw's patch matrix: the weight flattened to
        [320, Cin*9] and zero-padded to whole 64-wide K blocks (4 channels: 36 -> 64; 9 channels: 81 -> 128), like
        every other GEMM caller (none runs a partial K block)."""
        w_in = self.conv_in.weight.detach()
        co, ci = w_in.shape[0], w_in.shape[1]
        if ci != self.config.in_channels:
            raise IHError(f"{type(self).__name__}: config.in_channels = {self.config.in_channels} but conv_in.weight "
                          f"has {ci} input channels")
        self._w_in = torch.zeros((co, 64 if ci == 4 else 128), dtype=w_in.dtype, device=w_in.device)
        self._w_in[:, : ci * 9] = w_in.reshape(co, ci * 9)

    # ------------------------------------------------------------------------------------------------------------
    def prepare_conditioning(self, encoder_hidden_states: torch.Tensor, text_embeds: torch.Tensor,
                             time_ids: torch.Tensor) -> None:
        """Everything that does not depend on the step: cross-attention K/V of all attn2 layers (text and image
        tokens) and the text_time additional embedding."""
        cfg = self.config
        ehs = encoder_hidden_states
        B, L, _ = ehs.shape
        n_ip = next((p.num_tokens for p in self.attn_processors.values() if hasattr(p, "num_tokens")),
                    cfg.num_ip_tokens)
        n_text = L - n_ip
        text_only = ehs[:, :n_text].contiguous()
        self._text_only = text_only
        for name, attn in self._attn_modules():
            if attn.is_cross and hasattr(attn.processor, "prepare"):
                attn.processor.prepare(attn, ehs, text_only=text_only)
        if time_ids.numel() != B * cfg.num_time_ids:
            raise IHError(f"time_ids: {cfg.num_time_ids} micro-conditioning ids per image expected, got a tensor of shape "
                          f"{tuple(time_ids.shape)} for {B} images")
        tid = ops.sinusoid(time_ids.reshape(-1).float().contiguous(), cfg.addition_time_embed_dim, B * cfg.num_time_ids)
        add_in = torch.cat([text_embeds.to(torch.float16), tid.reshape(B, -1)], dim=-1).contiguous()
        h = ops.linear_small(add_in, self.add_embedding.linear_1.weight, self.add_embedding.linear_1.bias, act_out=True)
        buf = self._aug_bufs.get(B)                            # one buffer per batch size, never freed or moved
        if buf is None or buf.device != h.device:
            buf = torch.empty((B, cfg.time_embed_dim), dtype=torch.float16, device=h.device)
            self._aug_bufs[B] = buf
        aug = ops.linear_small(h, self.add_embedding.linear_2.weight, self.add_embedding.linear_2.bias, out=buf)
        self._aug = (self._aug_key(text_embeds, time_ids, B), aug)

    @staticmethod
    def _aug_key(text_embeds: torch.Tensor, time_ids: torch.Tensor, B: int):
        def ver(t):
            try:
                return t._version
            except RuntimeError:       # inference tensors do not track versions
                return -1
        return (text_embeds.data_ptr(), ver(text_embeds), time_ids.data_ptr(), ver(time_ids), B)

    def _ensure_conditioning(self, encoder_hidden_states, text_embeds, time_ids, B: int) -> None:
        if self._w_temb is None:
            raise IHError(f"{type(self).__name__}.finalize() has not been called")
        key = None if text_embeds is None else self._aug_key(text_embeds, time_ids, B)
        if self._aug is None or (key is not None and self._aug[0] != key):
            if text_embeds is None:
                raise IHError("forward() needs text_embeds/time_ids (or a prior prepare_conditioning())")
            self.prepare_conditioning(encoder_hidden_states, text_embeds, time_ids)

    def time_embeddings(self, timesteps: torch.Tensor, step: Optional[torch.Tensor], B: int) -> torch.Tensor:
        """-> temb_all [B, sum(Cout)]: every ResBlock's time_emb_proj(silu(emb)) in one launch."""
        cfg = self.config
        t_in = ops.sinusoid(timesteps, cfg.block_out_channels[0], B, step=step)
        h = ops.linear_small(t_in, self.time_embedding.linear_1.weight, self.time_embedding.linear_1.bias, act_out=True)
        emb = ops.linear_small(h, self.time_embedding.linear_2.weight, self.time_embedding.linear_2.bias,
                               addend=self._aug[1])
        return ops.linear_small(emb, self._w_temb, self._b_temb, act_in=True)


class UNet2DConditionModel(SDXLEncoderModel):
    """Native SDXL UNet. Build on the meta device + `load_state_dict(..., assign=True)` or via `from_state_dict`."""

    def __init__(self, cfg: UNetConfig):
        super().__init__()
        if cfg.in_channels not in (4, 9):
            raise IHError(f"UNet2DConditionModel: in_channels must be 4 (latents) or 9 (inpainting: latents | mask | "
                          f"masked-image latents), got {cfg.in_channels}")
        self.config = cfg
        boc = cfg.block_out_channels
        tl = cfg.transformer_layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], cfg.time_embed_dim)
        self.add_embedding = TimestepEmbedding(cfg.add_embed_in, cfg.time_embed_dim)
        downs = []
        ch = boc[0]
        for i, co in enumerate(boc):
            downs.append(DownBlock(cfg, ch, co, tl[i], add_down=i < len(boc) - 1))
            ch = co
        self.down_blocks = nn.ModuleList(downs)
        rev = list(reversed(boc))
        rtl = list(reversed(tl))
        ups = []
        prev = rev[0]
        for i, co in enumerate(rev):
            skip_ch = rev[min(i + 1, len(rev) - 1)]
            ups.append(UpBlock(cfg, prev, skip_ch, co, rtl[i], add_up=i < len(rev) - 1))
            prev = co
        self.up_blocks = nn.ModuleList(ups)
        self.mid_block = MidBlock(cfg, boc[-1], cfg.mid_depth)
        self.conv_norm_out = nn.GroupNorm(cfg.norm_num_groups, boc[0], eps=1e-5)
        self.conv_out = nn.Conv2d(boc[0], cfg.out_channels, 3, padding=1)

    def install_default_processors(self, scale: float = 1.0):
        """IPAdapter.set_ip_adapter (ip_adapter.py:99-125) for this UNet; IP weights are zero until loaded.  A UNet
        without image-prompt tokens (num_ip_tokens = 0, the refiner) gets diffusers' default instead: every
        cross-attention attends to all text tokens (CNAttnProcessor2_0 with num_tokens = 0, as on the ControlNet)."""
        from ip_adapter.attention_processor import AttnProcessor2_0, CNAttnProcessor2_0, IPAttnProcessor2_0
        cfg = self.config
        if cfg.num_ip_tokens == 0:
            procs = CNAttnProcessor2_0(num_tokens=0)
            self.set_attn_processor(procs)
            return self.attn_processors
        procs = {}
        dev = self.conv_in.weight.device
        for name, attn in self._attn_modules():
            if name.endswith("attn1"):
                procs[name + ".processor"] = AttnProcessor2_0()
            else:
                C = attn.to_q.weight.shape[0]
                with torch.device("meta"):
                    p = IPAttnProcessor2_0(C, cfg.cross_attention_dim, scale=scale, num_tokens=cfg.num_ip_tokens,
                                           skip=cfg.ip_target_substring not in name)
                p = p.to_empty(device=dev).half()
                for q in p.parameters():
                    q.data.zero_()
                    q.requires_grad_(False)
                procs[name + ".processor"] = p
        self.set_attn_processor(procs)
        return procs

    def _finalize_ends(self):
        # conv_in and conv_out run on the tensor-core GEMM: conv_in as in _pack_conv_in; conv_out weight tap-major with
        # Cout padded 4 -> 16
        self._pack_conv_in()
        w_out = ops.pack_conv3x3_weight(self.conv_out.weight.detach())            # [4, 9*320]
        self._w_out = torch.zeros((16, w_out.shape[1]), dtype=w_out.dtype, device=w_out.device)
        self._w_out[: w_out.shape[0]] = w_out
        self._b_out = torch.zeros((16,), dtype=w_out.dtype, device=w_out.device)
        self._b_out[: w_out.shape[0]] = self.conv_out.bias.detach()

    def _down_mid_with_adapter(self, x, temb_all, ehs, skips, adapter_residuals):
        """The down and mid blocks with T2I-Adapter features added at diffusers' points (see forward)."""
        if self.config.in_channels != 4:
            raise IHError("adapter_residuals: the T2I-Adapter runs with the 4-channel UNet only (diffusers has no SDXL "
                          "adapter pipeline for the 9-channel inpainting UNet)")
        feats, scale = adapter_residuals
        B, H, W, _ = x.shape
        require_adapter_shapes(self.config, H, W, [f.shape[1:] for f in feats])
        m = feats[0].shape[0]
        if any(f.shape[0] != m for f in feats) or B % m or scale.numel() < B // m:
            raise IHError(f"adapter_residuals: features of {[f.shape[0] for f in feats]} images and {scale.numel()} "
                          f"scales for a batch of {B}")
        pending = list(feats)

        def add(t: torch.Tensor) -> None:
            f = pending.pop(0)
            rows = m * f.shape[1] * f.shape[2]
            ops.controlnet_add_residuals([t] * (B // m), [f] * (B // m), scale, [r * rows for r in range(B // m)])

        for blk in self.down_blocks:
            if pending and blk.has_attn:
                x = blk(x, temb_all, ehs, skips, inject=add)
            else:
                x = blk(x, temb_all, ehs, skips)
                if pending:
                    add(x)                  # in place: the skip this block appended last is x itself
        x = self.mid_block(x, temb_all, ehs)
        if pending:                         # require_adapter_shapes: it has the mid block's shape
            add(x)
        return x

    def forward(self, sample: torch.Tensor, timesteps: torch.Tensor, encoder_hidden_states: torch.Tensor,
                text_embeds: Optional[torch.Tensor] = None, time_ids: Optional[torch.Tensor] = None,
                step: Optional[torch.Tensor] = None, cond: Optional[torch.Tensor] = None,
                controlnet_residuals=None, adapter_residuals=None) -> torch.Tensor:
        """sample NCHW fp16 [B,4,H,W]; timesteps fp32 device tensor ([B] values, or the whole schedule when `step`
        -- a device int32 index -- is given); returns noise prediction NCHW fp16.  The 9-channel inpainting UNet also
        takes `cond` NCHW fp16 [B,5,H,W] (mask | masked-image latents), which conv_in reads after the 4 latent channels;
        the 4-channel UNet takes no `cond`.

        `controlnet_residuals` = (ControlNetOutput, row offset in images): diffusers' down_block_additional_residuals
        and mid_block_additional_residual.  Residual k, times the output's scale[k], is added to skip k (9 of them) and
        to the mid-block output, into the rows of the images from the offset on (n in guess mode: the ControlNet ran on
        the conditional half only, the unconditional half gets nothing).  With a list of ControlNetOutputs (one per net
        of a Multi-ControlNet, one row offset for all) the nets' scaled residuals are summed in fp16 in list order and
        the sum is added, in one launch (ops.controlnet_add_residuals_multi).

        `adapter_residuals` = (features, scale): T2I-Adapter features, diffusers' down_intrablock_additional_residuals.
        features[k] is NHWC fp16 [m, h_k, w_k, C_k] with m dividing the batch (the features of one CFG half); scale is
        a device fp32 vector with at least batch / m entries, all the same value.  Feature k is added in place, as
        fp16(x + fp16(feature * scale)), to each group of m images at injection point k (adapter_targets): after a
        down block without cross-attention (its skip, the same tensor, sees the sum), after the last resnet /
        attention pair of one with it (before the skip is taken and the block downsamples), and a leftover feature
        after the mid block.  One launch per point; diffusers' single fp16(v * s) and fp16 add give the same bits."""
        if self._w_temb is None:
            raise IHError("UNet2DConditionModel.finalize() has not been called")
        B = sample.shape[0]
        n_cond = self.config.in_channels - sample.shape[1]
        if n_cond == 0 and cond is not None:
            raise IHError(f"UNet2DConditionModel: `sample` already has all {self.config.in_channels} input channels; "
                          "`cond` must be None")
        if n_cond > 0 and (cond is None or tuple(cond.shape) != (B, n_cond) + tuple(sample.shape[2:])):
            raise IHError(f"UNet2DConditionModel: the {self.config.in_channels}-channel UNet needs `cond` of shape "
                          f"{(B, n_cond) + tuple(sample.shape[2:])}, got {None if cond is None else tuple(cond.shape)}")
        require_latent_size(self.config, sample.shape[2], sample.shape[3])
        self._ensure_conditioning(encoder_hidden_states, text_embeds, time_ids, B)
        temb_all = self.time_embeddings(timesteps, step, B)
        Bs, _, Hs, Ws = sample.shape
        kpad = self._w_in.shape[1]
        a = ops.im2col3x3_nchw(sample, kpad) if cond is None else ops.im2col3x3_nchw_cat(sample, cond, kpad)
        x = ops.linear(a, self._w_in, self.conv_in.bias).reshape(Bs, Hs, Ws, -1)
        skips = [x]
        ehs = encoder_hidden_states
        if adapter_residuals is None:
            for blk in self.down_blocks:
                x = blk(x, temb_all, ehs, skips)
            x = self.mid_block(x, temb_all, ehs)
        else:
            x = self._down_mid_with_adapter(x, temb_all, ehs, skips, adapter_residuals)
        if controlnet_residuals is not None:
            # in place, and only here: the mid block has consumed skips[-1] (its input), and no skip is read again
            # before the up blocks pop them, so nothing sees a skip both before and after the addition
            cn, images = controlnet_residuals
            targets = skips + [x]
            for out in (cn if isinstance(cn, (list, tuple)) else [cn]):
                if len(out.residuals) != len(targets):
                    raise IHError(f"controlnet_residuals: {len(out.residuals)} residuals for {len(targets)} skip tensors")
            row0s = [images * (t.numel() // (t.shape[-1] * B)) for t in targets]
            if isinstance(cn, (list, tuple)):
                ops.controlnet_add_residuals_multi(targets, [o.residuals for o in cn], [o.scale for o in cn], row0s)
            else:
                ops.controlnet_add_residuals(targets, cn.residuals, cn.scale, row0s)
        for blk in self.up_blocks:
            x = blk(x, temb_all, ehs, skips)
        x = ops.groupnorm(x, self.conv_norm_out.weight, self.conv_norm_out.bias, groups=self.config.norm_num_groups,
                          eps=1e-5, silu=True)
        y16 = ops.conv3x3(x, self._w_out, self._b_out)
        return ops.nhwc_to_nchw(y16, self.config.out_channels)
