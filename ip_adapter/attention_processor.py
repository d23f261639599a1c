"""Attention processors with the reference's names, constructor arguments, state-dict keys and call protocol
(reference: ip_adapter/attention_processor.py:244-465), running on the sm_90a kernels of libimagharmony_sm90.so.

Protocol (attention_processor.py:364-371):  proc(attn, hidden_states, encoder_hidden_states=None,
attention_mask=None, temb=None) -> Tensor, with `attn` exposing heads / to_q / to_k / to_v / to_out.
Only the SDXL case of the reference is implemented (3-D hidden states, no mask, no spatial/group/cross norm,
no residual_connection, rescale 1.0) -- anything else raises instead of silently diverging.

Kernel-side differences that do not change results:
  * K/V of the encoder tokens are step-invariant; `prepare()` computes them once per generate() and the per-step call
    reuses them (the reference recomputes to_k/to_v/to_k_ip/to_v_ip every step, :410-411, :432-433).
  * text and image-prompt keys live in one [text ; ip] K/V buffer; the kernel runs the two softmaxes separately and a
    single PV MMA produces  SDPA_text + scale * SDPA_ip  (:423-450).
  * an optional `residual=` keyword fuses the block's `h + attn(...)` into the to_out GEMM epilogue.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from imagharmony_b200 import ops
from imagharmony_b200._lib import IHError


def _check_sdxl_case(attn, hidden_states, attention_mask):
    if hidden_states.dim() != 3:
        raise IHError("native processors implement the SDXL case: hidden_states must be [B, N, C]")
    if attention_mask is not None:
        raise IHError("attention_mask is not supported by the native processors (SDXL never passes one)")
    if getattr(attn, "spatial_norm", None) is not None or getattr(attn, "group_norm", None) is not None \
            or getattr(attn, "norm_cross", False) or getattr(attn, "residual_connection", False) \
            or getattr(attn, "rescale_output_factor", 1.0) != 1.0:
        raise IHError("native processors implement the SDXL case only (no spatial/group/cross norm, no residual "
                      "connection, rescale_output_factor == 1)")


def _cross_attention(attn, x, kv, B, N, Nk, C, *, n_ip=0, ip_scale=1.0, ln_stats=None, ln_eps=1e-5):
    """to_q + (decoupled) SDPA over the cached [K | V] rows: projection GEMM + attention kernel.
    Returns (q, output [B*N, C])."""
    if ln_stats is not None:
        (w, bias), ln = attn._ln, (ln_stats, ln_eps)              # norm2 folded into to_q
    else:
        w, bias, ln = attn.to_q.weight, None, None
    ops.prefetch_next(attn.to_out[0].weight)                      # L2 hint: the out projection follows the attention
    q = ops.linear(x, w, bias, ln=ln)
    return q, ops.attention(q, kv[:, :C], kv[:, C:], B, attn.heads, N, Nk, n_ip=n_ip, ip_scale=ip_scale)


class AttnProcessor2_0(torch.nn.Module):
    """Self-attention (and plain cross-attention) processor -- reference AttnProcessor2_0 (:244-332).

    Native extensions (keyword-only, used by imagharmony_b200.unet): `residual=` fuses the block's h + attn(...),
    `ln_stats=` means `hidden_states` are the RAW block input whose LayerNorm is folded into the q|k|v GEMM,
    `stats_out=` receives the row statistics of the output for the next folded LayerNorm."""

    supports_fused = True

    def __init__(self, hidden_size=None, cross_attention_dim=None):
        super().__init__()
        if not hasattr(F, "scaled_dot_product_attention"):   # kept for interface parity with :254-255
            raise ImportError("AttnProcessor2_0 requires PyTorch 2.0, to use it, please upgrade PyTorch to 2.0.")

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None,
                 *args, residual: Optional[torch.Tensor] = None, ln_stats: Optional[torch.Tensor] = None,
                 ln_eps: float = 1e-5, stats_out: Optional[torch.Tensor] = None, **kwargs):
        _check_sdxl_case(attn, hidden_states, attention_mask)
        B, N, C = hidden_states.shape
        H = attn.heads
        x = hidden_states.reshape(B * N, C)
        if encoder_hidden_states is None:
            ops.prefetch_next(attn.to_out[0].weight)                              # L2 hint for the launch after q|k|v
            if ln_stats is not None:
                w_c, c = attn._ln
                qkv = ops.linear(x, w_c, c, ln=(ln_stats, ln_eps))                # LayerNorm folded into q|k|v
            else:
                qkv = ops.linear(x, attn.fused_qkv_weight())                      # to_q | to_k | to_v in one GEMM
            o = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, H, N, N)
        else:
            Nk = encoder_hidden_states.shape[1]
            kv = ops.linear(encoder_hidden_states.reshape(B * Nk, -1), attn.fused_kv_weight())
            _, o = _cross_attention(attn, x, kv, B, N, Nk, C, ln_stats=ln_stats, ln_eps=ln_eps)
        res2d = None if residual is None else residual.reshape(B * N, C)
        ops.prefetch_next(getattr(attn, "_next_w", None))                         # weight of the GEMM that follows this block part
        out = ops.linear(o, attn.to_out[0].weight, attn.to_out[0].bias, residual=res2d,
                         stats_out=stats_out)                                     # :320 (+ fused h + ...)
        return out.reshape(B, N, C)


class IPAttnProcessor2_0(torch.nn.Module):
    """Decoupled image-prompt cross-attention -- reference IPAttnProcessor2_0 (:335-465).

    Owns `to_k_ip.weight` / `to_v_ip.weight` [hidden, cross_dim] (no bias, :361-362); public mutable attributes
    `scale`, `skip`, `num_tokens` exactly like the reference (set_scale mutates `scale`, ip_adapter.py:179-182).
    Native keyword extensions as in AttnProcessor2_0 (residual=, ln_stats=, ln_eps=, stats_out=).
    """

    supports_fused = True

    def __init__(self, hidden_size, cross_attention_dim=None, scale=1.0, num_tokens=4, skip=False):
        super().__init__()
        if not hasattr(F, "scaled_dot_product_attention"):
            raise ImportError("AttnProcessor2_0 requires PyTorch 2.0, to use it, please upgrade PyTorch to 2.0.")
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale
        self.num_tokens = num_tokens
        self.skip = skip
        self.to_k_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.to_v_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.keep_attn_map = False     # the reference's attn_map side effect (:443-444) has no consumer: opt-in
        self._kv = None                # (key, kv tensor [B*Nk, 2C], Nk, n_ip) of the last prepare()
        self._kv_bufs = {}             # (rows, 2C) -> buffer; kept until invalidate(): captured CUDA graphs point at them
        self._w_kv_ip = None

    # -- step-invariant K/V -------------------------------------------------------------------------------------
    def _ip_weight(self):
        w = self._w_kv_ip
        if w is None or w.device != self.to_k_ip.weight.device or w.dtype != self.to_k_ip.weight.dtype:
            w = torch.cat([self.to_k_ip.weight.detach(), self.to_v_ip.weight.detach()], dim=0).contiguous()
            self._w_kv_ip = w
        return w

    def invalidate(self):
        """Drop the cached K/V (weights changed).  Graphs captured against the old buffers are stale afterwards: the
        owner (UNet2DConditionModel.finalize / set_attn_processor) bumps its graph epoch so DenoiseEngine re-captures."""
        self._kv = None
        self._kv_bufs = {}
        self._w_kv_ip = None

    def _kv_buffer(self, rows: int, cols: int, like: torch.Tensor) -> torch.Tensor:
        """One K/V buffer per shape, never freed or moved while graphs may reference it (n=1 -> n=4 -> n=1 sequences of
        two-phase PNS / generate(num_samples=...) replay each shape's graph against that shape's own buffer)."""
        buf = self._kv_bufs.get((rows, cols))
        if buf is None or buf.device != like.device:
            buf = torch.empty((rows, cols), dtype=torch.float16, device=like.device)
            self._kv_bufs[(rows, cols)] = buf
        return buf

    @staticmethod
    def _key(ehs: torch.Tensor):
        try:
            version = ehs._version
        except RuntimeError:           # inference tensors do not track versions
            version = -1
        return (ehs.data_ptr(), tuple(ehs.shape), version)

    def prepare(self, attn, encoder_hidden_states: torch.Tensor, text_only: Optional[torch.Tensor] = None):
        """Compute and cache K/V for these encoder tokens: [text ; ip] for active layers, text only when skip."""
        ehs = encoder_hidden_states
        B, L, D = ehs.shape
        n_text = L - self.num_tokens                                             # :402
        C = self.hidden_size
        w_kv = attn.fused_kv_weight()
        if self.skip:
            if text_only is None:
                text_only = ehs[:, :n_text].contiguous()
            kv = ops.linear(text_only.reshape(B * n_text, D), w_kv,
                            out=self._kv_buffer(B * n_text, 2 * C, ehs))         # :410-411
            self._kv = (self._key(ehs), kv, n_text, 0)
        else:
            kv = ops.linear(ehs.reshape(B * L, D), w_kv, out=self._kv_buffer(B * L, 2 * C, ehs))   # text rows: to_k / to_v
            ip = ehs[:, n_text:].contiguous().reshape(B * self.num_tokens, D)
            kv_ip = ops.linear(ip, self._ip_weight())                            # :432-433 to_k_ip / to_v_ip
            kv.view(B, L, 2 * C)[:, n_text:] = kv_ip.view(B, self.num_tokens, 2 * C)
            self._kv = (self._key(ehs), kv, L, self.num_tokens)
        return self._kv

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None,
                 residual: Optional[torch.Tensor] = None, ln_stats: Optional[torch.Tensor] = None,
                 ln_eps: float = 1e-5, stats_out: Optional[torch.Tensor] = None):
        _check_sdxl_case(attn, hidden_states, attention_mask)
        if encoder_hidden_states is None:
            raise IHError("IPAttnProcessor2_0 needs encoder_hidden_states (it is installed on attn2 only)")
        B, N, C = hidden_states.shape
        cached = self._kv
        if cached is None or cached[0] != self._key(encoder_hidden_states):
            cached = self.prepare(attn, encoder_hidden_states)
        _, kv, Nk, n_ip = cached
        x = hidden_states.reshape(B * N, C)
        want_map = self.keep_attn_map and not self.skip
        q, o = _cross_attention(attn, x, kv, B, N, Nk, C, n_ip=n_ip, ip_scale=float(self.scale), ln_stats=ln_stats,
                                ln_eps=ln_eps)                                    # :396, :423-450
        if want_map:
            k_ip = kv.view(B, Nk, 2 * C)[:, Nk - n_ip:, :C].reshape(B, n_ip, attn.heads, 64).permute(0, 2, 1, 3)
            qh = q.reshape(B, N, attn.heads, 64).permute(0, 2, 1, 3)
            self.attn_map = qh @ k_ip.to(qh.dtype).transpose(-2, -1).softmax(dim=-1)   # :443-444 (diagnostic only)
        res2d = None if residual is None else residual.reshape(B * N, C)
        ops.prefetch_next(getattr(attn, "_next_w", None))
        out = ops.linear(o, attn.to_out[0].weight, attn.to_out[0].bias, residual=res2d, stats_out=stats_out)   # :453
        return out.reshape(B, N, C)


class CNAttnProcessor2_0(AttnProcessor2_0):
    """The processor IPAdapter installs on a ControlNet -- reference CNAttnProcessor2_0 (:534-621): self-attention as
    AttnProcessor2_0, cross-attention over the text tokens only (the last `num_tokens` image-prompt tokens are
    dropped, :570-571), so the ControlNet never sees the image prompt.  Like the reference it is one object installed
    on every attention module.  Cross-attention is delegated to one text-only IPAttnProcessor2_0 (skip=True) per
    module, which caches that module's step-invariant text K/V; its unused image-prompt weights stay on the meta
    device (no memory), and it is not a registered submodule, so this processor has no parameters."""

    def __init__(self, num_tokens=4):
        super().__init__()
        self.num_tokens = num_tokens
        self._text = {}                # id(attn) -> IPAttnProcessor2_0(skip=True) of that attention module

    def _text_processor(self, attn) -> IPAttnProcessor2_0:
        p = self._text.get(id(attn))
        if p is None:
            C, D = attn.to_q.weight.shape[0], attn.to_k.weight.shape[1]
            with torch.device("meta"):
                p = IPAttnProcessor2_0(C, D, num_tokens=self.num_tokens, skip=True)
            self._text[id(attn)] = p
        return p

    def invalidate(self):
        """Drop the cached K/V (weights changed); the owner bumps its graph epoch."""
        self._text = {}

    def prepare(self, attn, encoder_hidden_states: torch.Tensor, text_only: Optional[torch.Tensor] = None):
        return self._text_processor(attn).prepare(attn, encoder_hidden_states, text_only=text_only)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None,
                 residual: Optional[torch.Tensor] = None, ln_stats: Optional[torch.Tensor] = None,
                 ln_eps: float = 1e-5, stats_out: Optional[torch.Tensor] = None):
        if encoder_hidden_states is None:
            return super().__call__(attn, hidden_states, None, attention_mask, temb, residual=residual,
                                    ln_stats=ln_stats, ln_eps=ln_eps, stats_out=stats_out)
        return self._text_processor(attn)(attn, hidden_states, encoder_hidden_states, attention_mask, temb,
                                          residual=residual, ln_stats=ln_stats, ln_eps=ln_eps, stats_out=stats_out)


# names the reference exports for torch < 2 are intentionally absent (out of scope, SURVEY.md section 2)
AttnProcessor = AttnProcessor2_0
IPAttnProcessor = IPAttnProcessor2_0
CNAttnProcessor = CNAttnProcessor2_0

# `from ip_adapter.attention_processor import Cross_Attention` (train.py:32): HarmonyAttention's attention block
# (attention_processor.py:12-56) lives with the adapter modules
from imagharmony_b200.adapter import Cross_Attention  # noqa: E402,F401
