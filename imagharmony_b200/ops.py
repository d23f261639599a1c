"""One Python function per C-ABI entry point of libimagharmony_sm90.so (include/ih_api.h).

Tensors are torch CUDA fp16; PyTorch is only used for device memory and the current stream. No op has a
PyTorch/CPU fallback: a CPU tensor or a missing library raises.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import IH_SOLVER_DPMPP_2M, IH_SOLVER_UNIPC_BH2, IH_UNIPC_COEFFS, IHError, check

EPI_NONE, EPI_GEGLU, EPI_SILU, EPI_GELU, EPI_QUICK_GELU, EPI_RELU = 0, 1, 2, 4, 8, 16
TILE_PINGPONG = 1   # IH_TILE_PINGPONG: linear(tile_n=TILE_PINGPONG) forces the ping-pong GEMM kernel


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, name: str, dtype=torch.float16) -> None:
    if not t.is_cuda:
        raise IHError(f"{name}: expected a CUDA tensor (the sm_90a path has no CPU fallback)")
    if t.dtype != dtype:
        raise IHError(f"{name}: expected dtype {dtype}, got {t.dtype}")


def _rows(t: torch.Tensor, name: str) -> int:
    """Row stride (elements) of a 2-D view whose last dim is contiguous."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise IHError(f"{name}: expected a 2-D tensor with contiguous last dim, got shape {tuple(t.shape)} "
                      f"strides {t.stride()}")
    return t.stride(0)


def launch_count() -> int:
    return int(_lib.load().ih_launch_count())


def launch_count_reset() -> None:
    _lib.load().ih_launch_count_reset()


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
           residual: Optional[torch.Tensor] = None, rowbias: Optional[torch.Tensor] = None,
           rows_per_group: int = 0, geglu: bool = False, silu: bool = False, gelu: bool = False,
           out: Optional[torch.Tensor] = None, tile_n: int = 0, ln=None,
           stats_out: Optional[torch.Tensor] = None, quick_gelu: bool = False, alpha: float = 1.0,
           relu: bool = False) -> torch.Tensor:
    """out = epi(x @ w.T + bias + rowbias[row // rows_per_group]) + residual ; x [M,K], w [N,K] (nn.Linear layout).
    `relu=True`: out = relu(alpha * x @ w.T + bias + residual), the ReLU after the residual (IH_EPI_RELU); it takes no
    other activation, rowbias, ln, stats_out or tile_n.
    `tile_n`: 0 lets the library choose; else 64 / 128 / 160 / 192 / 256 output columns per tile, or with `geglu`
    128 / 192 / 256 weight rows per tile (value and gate halves: 64 / 96 / 128 outputs).  `tile_n=TILE_PINGPONG`
    forces the ping-pong kernel (bias, ln and geglu only), which the library's choice takes where it is faster.

    LayerNorm folding: `stats_out` (float32 [ceil(N/64), M, 2]) receives per-row (sum, sumsq) of the stored values as
    partial sums whose total over slots is the row's; `ln=(stats, eps)` makes this GEMM consume RAW rows `x` with the gamma-scaled, row-centred weight and
    the constant vector of fold_layernorm (passed as `w`, `bias`) and apply rstd * acc + bias in the epilogue."""
    lib = _lib.load()
    _req(x, "x"); _req(w, "w")
    M, K = x.shape
    N = w.shape[0]
    if w.shape[1] != K or not w.is_contiguous():
        raise IHError(f"linear: weight must be contiguous [N,{K}], got {tuple(w.shape)}")
    n_out = N // 2 if geglu else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float16, device=x.device)
    ldr = _rows(residual, "residual") if residual is not None else 0
    ldrb = _rows(rowbias, "rowbias") if rowbias is not None else 0
    epi = ((EPI_GEGLU if geglu else 0) | (EPI_SILU if silu else 0) | (EPI_GELU if gelu else 0)
           | (EPI_QUICK_GELU if quick_gelu else 0))
    if relu:
        if epi:
            raise IHError("linear: relu cannot be combined with geglu / silu / gelu / quick_gelu")
        epi = EPI_RELU
    if alpha != 1.0 or relu:
        # out = epi(alpha * x w^T + bias) + residual (ih_gemm_scaled_f16: the VAE decoder's scaled residual stream), or
        # relu(alpha * x w^T + bias + residual)
        if ln is not None or stats_out is not None or rowbias is not None or tile_n:
            raise IHError("linear: alpha != 1 / relu cannot be combined with ln / stats_out / rowbias / tile_n")
        rc = lib.ih_gemm_scaled_f16(x.data_ptr(), _rows(x, "x"), w.data_ptr(), _p(bias), _p(residual), ldr, out.data_ptr(),
                                    _rows(out, "out"), M, N, K, epi, float(alpha), _stream())
        check(rc, "ih_gemm_scaled_f16")
        return out
    if ln is None and stats_out is None:
        rc = lib.ih_gemm_f16(x.data_ptr(), _rows(x, "x"), w.data_ptr(), _p(bias), _p(rowbias), rows_per_group, ldrb,
                             _p(residual), ldr, out.data_ptr(), _rows(out, "out"), M, N, K, epi, tile_n, _stream())
        check(rc, "ih_gemm_f16")
        return out
    ln_stats = None
    ln_slabs, ln_eps = 0, 0.0
    if ln is not None:
        ln_stats, ln_eps = ln
        _req(ln_stats, "ln_stats", torch.float32)
        if ln_stats.dim() != 3 or ln_stats.shape[1] != M or ln_stats.shape[-1] != 2 or not ln_stats.is_contiguous():
            raise IHError("linear: ln statistics must be contiguous [slabs, M, 2]")
        if ln_stats.shape[0] != (K + 63) // 64:
            raise IHError(f"linear: ln statistics cover {ln_stats.shape[0]} slabs, K={K} needs {(K + 63) // 64}")
        ln_slabs = ln_stats.shape[0]
    if stats_out is not None:
        _req(stats_out, "stats_out", torch.float32)
        if tuple(stats_out.shape) != ((n_out + 63) // 64, M, 2) or not stats_out.is_contiguous():
            raise IHError(f"linear: stats_out must be contiguous float32 [{(n_out + 63) // 64}, {M}, 2]")
    rc = lib.ih_gemm_ln_f16(x.data_ptr(), _rows(x, "x"), w.data_ptr(), _p(bias), _p(rowbias), rows_per_group, ldrb,
                            _p(residual), ldr, out.data_ptr(), _rows(out, "out"), M, N, K, epi, tile_n, _p(ln_stats),
                            ln_slabs, float(ln_eps), _p(stats_out), _stream())
    check(rc, "ih_gemm_ln_f16")
    return out


def prefetch_next(w: Optional[torch.Tensor]) -> None:
    """Hint for the NEXT linear / conv3x3 call: while it runs, pull `w` (the weight of the launch after it) into L2."""
    if w is not None and w.is_cuda:
        _lib.load().ih_gemm_prefetch_next(w.data_ptr(), w.numel() * w.element_size())


def _round_rows_zero_sum(w: torch.Tensor, passes: int = 32) -> torch.Tensor:
    """fp16 rounding of fp64 rows that each sum to zero, keeping every fp16 row sum at zero.

    Round-to-nearest leaves a random-walk row sum (about 2e-4 for 1280 weights of scale 1280^-1/2).  The fold multiplies
    that sum by mean(x) * rstd(x), so its error would grow linearly with |mean| / std.  Each pass moves elements one fp16
    step toward the residual's sign, cheapest first, as long as the steps taken fit in the residual.  The first stage
    only moves elements that were rounded away from their exact value in that direction (they stay between its two
    fp16 neighbours); it leaves residuals of about 3e-7, which the second stage removes with the finest steps of the
    row, wherever they are.  The elementwise error stays that of round-to-nearest."""
    h = w.to(torch.float16)
    for between in (True, False):
        for _ in range(passes):
            r = h.double().sum(dim=1, keepdim=True)       # exact: fp16 values summed in fp64
            toward = torch.where(r > 0, float("-inf"), float("inf")).to(torch.float16).expand_as(h)
            alt = torch.nextafter(h, toward)
            step = (h.double() - alt.double()).abs()
            fits = (step <= r.abs()) & (r != 0)
            if between:
                fits &= (h.double() - w) * r > 0
            if not bool(fits.any()):
                break
            cost = torch.where(fits, (alt.double() - w).abs() - (h.double() - w).abs(), float("inf"))
            order = cost.argsort(dim=1)
            fits_sorted = fits.gather(1, order)
            cum = torch.cumsum(torch.where(fits_sorted, step.gather(1, order), 0.0), dim=1)
            take = torch.zeros_like(fits).scatter(1, order, fits_sorted & (cum <= r.abs()))
            h = torch.where(take, alt, h)
    return h


def fold_layernorm(w: torch.Tensor, bias: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor):
    """LayerNorm(x) @ w.T + bias == rstd(x) * (x @ w_c.T) + c with
       w_c[n, k] = w[n, k] gamma[k] - mean_k(w[n, :] gamma)   (rows centred: x @ w_c.T = (x - mean(x)) @ (w gamma).T)
       c[n]      = sum_k beta[k] w[n, k] + bias[n].
    w_c is rounded to fp16 so that its rows still sum to exactly zero (_round_rows_zero_sum): the mean of x then drops
    out of x @ w_c.T up to fp32 accumulation, whatever |mean| / std.
    Returns (w_c, c) in fp16 for ops.linear(x_raw, w_c, c, ln=(row statistics of x_raw, eps))."""
    w_g = w.double() * gamma.double()[None, :]
    w_c = _round_rows_zero_sum(w_g - w_g.mean(dim=1, keepdim=True)).contiguous()
    c = w.double() @ beta.double()
    if bias is not None:
        c = c + bias.double()
    return w_c, c.to(torch.float16).contiguous()


def conv3x3(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
            rowbias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None, stride: int = 1,
            out: Optional[torch.Tensor] = None, tile_n: int = 0, alpha: float = 1.0, shortcut=None,
            relu: bool = False) -> torch.Tensor:
    """3x3 conv, pad 1. x NHWC [B,H,W,Cin]; w_packed [Cout, 9*Cin] (see pack_conv3x3_weight); rowbias [B, >=Cout].
    `relu=True`: out = relu(alpha * conv(x) + bias + residual), the ReLU after the residual (IH_EPI_RELU).
    `shortcut=(s0, s1 | None)`: fused 1x1 shortcut conv over the channel concat of the NHWC tensors s0 [, s1]; then
    w_packed is [Cout, 9*Cin + C(s0) + C(s1)] (3x3 taps followed by the shortcut weight), see ih_conv2d_shortcut_f16."""
    lib = _lib.load()
    _req(x, "x"); _req(w_packed, "w")
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    if shortcut is not None:
        s0, s1 = shortcut
        c0, c1 = s0.shape[-1], (0 if s1 is None else s1.shape[-1])
        _req(s0, "shortcut[0]")
        if s1 is not None:
            _req(s1, "shortcut[1]")
        if (stride != 1 or residual is not None or alpha != 1.0 or relu or tile_n or not x.is_contiguous()
                or not s0.is_contiguous()
                or (s1 is not None and not s1.is_contiguous()) or tuple(s0.shape[:3]) != (B, H, W)
                or (s1 is not None and tuple(s1.shape[:3]) != (B, H, W)) or not w_packed.is_contiguous()
                or w_packed.shape[1] != 9 * Cin + c0 + c1):
            raise IHError("conv3x3(shortcut=): stride 1, no residual / alpha / relu / tile_n, contiguous NHWC sources of the same "
                          "spatial size and w_packed [Cout, 9*Cin + C0 + C1] required")
        if out is None:
            out = torch.empty((B, H, W, Cout), dtype=torch.float16, device=x.device)
        ldrb = _rows(rowbias, "rowbias") if rowbias is not None else 0
        rc = lib.ih_conv2d_shortcut_f16(x.data_ptr(), w_packed.data_ptr(), _p(bias), _p(rowbias), ldrb, s0.data_ptr(), c0,
                                        _p(s1), c1, out.data_ptr(), B, H, W, Cin, Cout, _stream())
        check(rc, "ih_conv2d_shortcut_f16")
        return out
    if not x.is_contiguous() or not w_packed.is_contiguous() or w_packed.shape[1] != 9 * Cin:
        raise IHError("conv3x3: x must be contiguous NHWC and w_packed [Cout, 9*Cin]")
    Ho, Wo = H // stride, W // stride
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), dtype=torch.float16, device=x.device)
    ldrb = _rows(rowbias, "rowbias") if rowbias is not None else 0
    if residual is not None and (not residual.is_contiguous() or residual.shape != out.shape):
        raise IHError("conv3x3: residual must be contiguous and shaped like the output")
    if alpha != 1.0 or relu:
        if rowbias is not None or tile_n:
            raise IHError("conv3x3: alpha != 1 / relu cannot be combined with rowbias / tile_n")
        rc = lib.ih_conv2d_scaled_f16(x.data_ptr(), w_packed.data_ptr(), _p(bias), _p(residual), out.data_ptr(), B, H, W,
                                      Cin, Cout, stride, float(alpha), _stream(), EPI_RELU if relu else EPI_NONE)
        check(rc, "ih_conv2d_scaled_f16")
        return out
    rc = lib.ih_conv2d_f16(x.data_ptr(), w_packed.data_ptr(), _p(bias), _p(rowbias), ldrb, _p(residual),
                           out.data_ptr(), B, H, W, Cin, Cout, 3, stride, tile_n, _stream())
    check(rc, "ih_conv2d_f16")
    return out


def conv3x3_down(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
                 out: Optional[torch.Tensor] = None, tile_n: int = 0, alpha: float = 1.0) -> torch.Tensor:
    """alpha * conv3x3(F.pad(x, (0, 1, 0, 1)), stride 2, pad 0) + bias: the VAE encoder's Downsample2D.  x NHWC
    [B, H, W, Cin] with H, W even; w_packed [Cout, 9*Cin]; returns [B, H/2, W/2, Cout]."""
    lib = _lib.load()
    _req(x, "x"); _req(w_packed, "w")
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    if not x.is_contiguous() or not w_packed.is_contiguous() or w_packed.shape[1] != 9 * Cin:
        raise IHError("conv3x3_down: x must be contiguous NHWC and w_packed [Cout, 9*Cin]")
    if out is None:
        out = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.float16, device=x.device)
    rc = lib.ih_conv2d_down_f16(x.data_ptr(), w_packed.data_ptr(), _p(bias), out.data_ptr(), B, H, W, Cin, Cout, tile_n,
                                float(alpha), _stream())
    check(rc, "ih_conv2d_down_f16")
    return out


def vae_posterior_noise(moments: torch.Tensor, eps: torch.Tensor, noise: torch.Tensor, channels: int,
                        scaling_factor: float, sigma: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Image-to-image initial latents (ih_vae_posterior_noise_f16): moments NHWC [Bm, h, w, >= 2*channels] fp16, eps
    NCHW [Be, channels, h, w] fp32 or fp16, noise NCHW [B, channels, h, w] fp16 -> NCHW fp16 [B, channels, h, w];
    image b uses moments[b % Bm] and eps[b % Be]."""
    lib = _lib.load()
    _req(moments, "moments"); _req(noise, "noise")
    if eps.dtype not in (torch.float32, torch.float16):
        raise IHError(f"vae_posterior_noise: eps must be float32 or float16, got {eps.dtype}")
    _req(eps, "eps", eps.dtype)
    Bm, h, w, ldc = moments.shape
    B = noise.shape[0]
    if (not (moments.is_contiguous() and eps.is_contiguous() and noise.is_contiguous())
            or tuple(noise.shape) != (B, channels, h, w) or tuple(eps.shape[1:]) != (channels, h, w)):
        raise IHError(f"vae_posterior_noise: contiguous eps [*, {channels}, {h}, {w}] and noise [B, {channels}, {h}, {w}] "
                      "required")
    if out is None:
        out = torch.empty((B, channels, h, w), dtype=torch.float16, device=moments.device)
    rc = lib.ih_vae_posterior_noise_f16(moments.data_ptr(), ldc, eps.data_ptr(), int(eps.dtype == torch.float32),
                                        noise.data_ptr(), out.data_ptr(), B, Bm, eps.shape[0], h * w, channels,
                                        float(scaling_factor), float(sigma), _stream())
    check(rc, "ih_vae_posterior_noise_f16")
    return out


def pack_conv3x3_weight(w_oihw: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, 3, 3] (nn.Conv2d) -> [Cout, 9*Cin] tap-major, the layout ih_conv2d_f16 expects."""
    Cout, Cin, kh, kw = w_oihw.shape
    assert kh == 3 and kw == 3
    return w_oihw.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()


_attn_ws = {}
_ws_generation = 0


def workspace_generation() -> int:
    """Bumped whenever a persistent scratch buffer (attention KV-split parts, GroupNorm statistics) is re-allocated.
    A CUDA graph captured under an older generation may hold a pointer to freed memory: DenoiseEngine compares this
    number with the one it recorded at capture time and re-captures instead of replaying a stale graph."""
    return _ws_generation


def _bump_generation() -> None:
    global _ws_generation
    _ws_generation += 1


def _attn_workspace(device, need: int) -> Optional[torch.Tensor]:
    """Persistent grow-only scratch for the KV-split self-attention parts (one per device; calls are stream-ordered)."""
    if need <= 0:
        return None
    ws = _attn_ws.get(device)
    if ws is None or ws.numel() < need:
        if torch.cuda.is_current_stream_capturing():
            raise IHError("attention workspace must be created before CUDA-graph capture (run one warm-up step)")
        had = ws is not None
        ws = torch.zeros(max(need, 16 << 20), dtype=torch.uint8, device=device)   # arrival counters start at zero
        _attn_ws[device] = ws
        if had:
            _bump_generation()
    return ws


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, H: int, Nq: int, Nk: int, *,
              n_ip: int = 0, ip_scale: float = 1.0, out: Optional[torch.Tensor] = None,
              kv_split: bool = True) -> torch.Tensor:
    """q [B*Nq, >=H*64] / k, v [B*Nk, >=H*64] 2-D views (row stride arbitrary); returns [B*Nq, H*64].
    kv_split=False withholds the workspace, i.e. every query tile is processed whole."""
    lib = _lib.load()
    _req(q, "q"); _req(k, "k"); _req(v, "v")
    if out is None:
        out = torch.empty((B * Nq, H * 64), dtype=torch.float16, device=q.device)
    ws = _attn_workspace(q.device, int(lib.ih_attention_workspace_bytes(B, H, Nq, Nk, n_ip))) if kv_split else None
    rc = lib.ih_attention_ws_f16(q.data_ptr(), _rows(q, "q"), k.data_ptr(), _rows(k, "k"), v.data_ptr(),
                                 _rows(v, "v"), out.data_ptr(), _rows(out, "out"), B, H, Nq, Nk, n_ip,
                                 float(ip_scale), _p(ws), 0 if ws is None else ws.numel(), _stream())
    check(rc, "ih_attention_ws_f16")
    return out


_gn_ws = {}


def _gn_workspace(device, B: int, groups: int) -> torch.Tensor:
    """Persistent zero-initialised statistics workspace (one per device; GroupNorm calls are stream-ordered)."""
    need = int(_lib.load().ih_groupnorm_workspace_bytes(B, groups))
    ws = _gn_ws.get(device)
    if ws is None or ws.numel() < need:
        if torch.cuda.is_current_stream_capturing():
            raise IHError("groupnorm workspace must be created before CUDA-graph capture (run one warm-up step)")
        had = ws is not None
        ws = torch.zeros(max(need, 1 << 20), dtype=torch.uint8, device=device)
        _gn_ws[device] = ws
        if had:
            _bump_generation()
    return ws


def groupnorm(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, x1: Optional[torch.Tensor] = None,
              groups: int = 32, eps: float = 1e-5, silu: bool = False, out: Optional[torch.Tensor] = None,
              ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm over NHWC x0 [B,H,W,C0] (optionally concatenated with x1 [B,H,W,C1] on channels)."""
    lib = _lib.load()
    _req(x0, "x0")
    B, H, W, C0 = x0.shape
    C1 = 0 if x1 is None else x1.shape[-1]
    if not x0.is_contiguous() or (x1 is not None and not x1.is_contiguous()):
        raise IHError("groupnorm: inputs must be contiguous NHWC")
    if out is None:
        out = torch.empty((B, H, W, C0 + C1), dtype=torch.float16, device=x0.device)
    if ws is None:
        ws = _gn_workspace(x0.device, B, groups)
    rc = lib.ih_groupnorm_f16(x0.data_ptr(), C0, _p(x1), C1, gamma.data_ptr(), beta.data_ptr(), out.data_ptr(),
                              ws.data_ptr(), B, H * W, groups, float(eps), int(silu), _stream())
    check(rc, "ih_groupnorm_f16")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, "x")
    if not x.is_contiguous():
        raise IHError("layernorm: x must be contiguous")
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    rc = lib.ih_layernorm_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), rows, C, float(eps),
                              _stream())
    check(rc, "ih_layernorm_f16")
    return out


def linear_small(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act_in: bool = False,
                 act_out: bool = False, addend: Optional[torch.Tensor] = None, out_scale: float = 1.0,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Small-M (<= 8 rows) linear with optional SiLU on the input and/or output and an optional fp16 addend."""
    lib = _lib.load()
    _req(x, "x"); _req(w, "w")
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float16, device=x.device)
    if M > 64:
        raise IHError(f"linear_small: M={M} > 64 rows; use ops.linear")
    ld_add = _rows(addend, "addend") if addend is not None else 0
    rc = lib.ih_linear_small_f16(x.data_ptr(), _rows(x, "x"), w.data_ptr(), _p(bias), _p(addend), ld_add,
                                 out.data_ptr(), _rows(out, "out"), M, N, K, int(act_in), int(act_out),
                                 float(out_scale), _stream())
    check(rc, "ih_linear_small_f16")
    return out


def attention_small(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, H: int, Nq: int, Nk: int, dqk: int,
                    dv: int, scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """CUDA-core attention for odd head sizes / few queries: q [B*Nq, H*dqk], k [B*Nk, H*dqk], v [B*Nk, H*dv]."""
    lib = _lib.load()
    _req(q, "q"); _req(k, "k"); _req(v, "v")
    if out is None:
        out = torch.empty((B * Nq, H * dv), dtype=torch.float16, device=q.device)
    rc = lib.ih_attention_small_f16(q.data_ptr(), _rows(q, "q"), k.data_ptr(), _rows(k, "k"), v.data_ptr(),
                                    _rows(v, "v"), out.data_ptr(), _rows(out, "out"), B, H, Nq, Nk, dqk, dv,
                                    float(scale), _stream())
    check(rc, "ih_attention_small_f16")
    return out


def attention_generic(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, H: int, Nq: int, Nk: int, dqk: int,
                      dv: int, scale: float, causal: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(q k^T * scale (+ causal mask)) v for any head dims that are multiples of 8 (CLIP towers: 64 causal,
    104 for ViT-bigG): q [B*Nq, >=H*dqk], k [B*Nk, >=H*dqk], v [B*Nk, >=H*dv] 2-D views."""
    lib = _lib.load()
    _req(q, "q"); _req(k, "k"); _req(v, "v")
    if out is None:
        out = torch.empty((B * Nq, H * dv), dtype=torch.float16, device=q.device)
    rc = lib.ih_attention_generic_f16(q.data_ptr(), _rows(q, "q"), k.data_ptr(), _rows(k, "k"), v.data_ptr(),
                                      _rows(v, "v"), out.data_ptr(), _rows(out, "out"), B, H, Nq, Nk, dqk, dv,
                                      float(scale), int(causal), _stream())
    check(rc, "ih_attention_generic_f16")
    return out


def embed_tokens(ids: torch.Tensor, tok_emb: torch.Tensor, pos_emb: torch.Tensor,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """ids int32 [B, T] (device) -> tok_emb[ids] + pos_emb[:T]  as [B*T, C] fp16."""
    lib = _lib.load()
    _req(ids, "ids", torch.int32); _req(tok_emb, "tok_emb"); _req(pos_emb, "pos_emb")
    B, T = ids.shape
    C = tok_emb.shape[1]
    if not (ids.is_contiguous() and tok_emb.is_contiguous() and pos_emb.is_contiguous()) or pos_emb.shape[0] < T:
        raise IHError("embed_tokens: contiguous ids / tables and pos_emb with >= T rows required")
    if out is None:
        out = torch.empty((B * T, C), dtype=torch.float16, device=ids.device)
    check(lib.ih_embed_tokens_f16(ids.data_ptr(), tok_emb.data_ptr(), pos_emb.data_ptr(), out.data_ptr(), B * T, T, C,
                                  tok_emb.shape[0], _stream()), "ih_embed_tokens_f16")
    return out


def resize_patchify(img: torch.Tensor, size: int, patch: int, kpad: int, mean, std,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """img NCHW fp16 in [-1, 1] -> area-averaged size x size, [0,1], (v - mean) / std, as patch rows
    [B * (size/patch)^2, kpad] with k = c*patch^2 + py*patch + px (zero padded)."""
    import ctypes
    lib = _lib.load()
    _req(img, "img")
    B, C, H, W = img.shape
    if not img.is_contiguous():
        raise IHError("resize_patchify: contiguous NCHW image required")
    g = size // patch
    if out is None:
        out = torch.empty((B * g * g, kpad), dtype=torch.float16, device=img.device)
    m3 = (ctypes.c_float * 3)(*[float(x) for x in mean])
    s3 = (ctypes.c_float * 3)(*[float(x) for x in std])
    check(lib.ih_resize_patchify_f16(img.data_ptr(), out.data_ptr(), B, C, H, W, size, patch, kpad, m3, s3, _stream()),
          "ih_resize_patchify_f16")
    return out


def add_bcast(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """a + b where b is broadcast over the leading elements of a (a.numel() % b.numel() == 0), contiguous fp16."""
    lib = _lib.load()
    _req(a, "a"); _req(b, "b")
    if not (a.is_contiguous() and b.is_contiguous()) or a.numel() % b.numel() != 0:
        raise IHError("add_bcast: contiguous tensors with a.numel() % b.numel() == 0 required")
    if out is None:
        out = torch.empty_like(a)
    check(lib.ih_add_bcast_f16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), b.numel(), _stream()),
          "ih_add_bcast_f16")
    return out


def mean_tokens(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[B, n, D] -> [B, D] mean over tokens."""
    lib = _lib.load()
    _req(x, "x")
    B, n, D = x.shape
    if not x.is_contiguous():
        raise IHError("mean_tokens: x must be contiguous")
    if out is None:
        out = torch.empty((B, D), dtype=torch.float16, device=x.device)
    check(lib.ih_mean_tokens_f16(x.data_ptr(), out.data_ptr(), B, n, D, _stream()), "ih_mean_tokens_f16")
    return out


def sinusoid(t: torch.Tensor, dim: int, n: int, *, step: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[n, dim] fp16 sinusoidal embedding of fp32 `t` (or of t[step] for every row when `step` is given)."""
    lib = _lib.load()
    _req(t, "t", torch.float32)
    if out is None:
        out = torch.empty((n, dim), dtype=torch.float16, device=t.device)
    rc = lib.ih_sinusoid_f16(t.data_ptr(), _p(step), out.data_ptr(), _rows(out, "out"), n, dim, _stream())
    check(rc, "ih_sinusoid_f16")
    return out


def upsample2x(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, "x")
    B, H, W, C = x.shape
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float16, device=x.device)
    check(lib.ih_upsample2x_f16(x.data_ptr(), out.data_ptr(), B, H, W, C, _stream()), "ih_upsample2x_f16")
    return out


def concat_channels(x0: torch.Tensor, x1: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x0, "x0"); _req(x1, "x1")
    C0, C1 = x0.shape[-1], x1.shape[-1]
    rows = x0.numel() // C0
    if out is None:
        out = torch.empty(tuple(x0.shape[:-1]) + (C0 + C1,), dtype=torch.float16, device=x0.device)
    check(lib.ih_concat_f16(x0.data_ptr(), C0, x1.data_ptr(), C1, out.data_ptr(), rows, _stream()), "ih_concat_f16")
    return out


def im2col3x3_nchw(x_nchw: torch.Tensor, kpad: int = 64, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[B, Cin, H, W] -> A [B*H*W, kpad] with k = ci*9 + ky*3 + kx (zero padded): conv_in as a tensor-core GEMM."""
    lib = _lib.load()
    _req(x_nchw, "x")
    B, Cin, H, W = x_nchw.shape
    if out is None:
        out = torch.empty((B * H * W, kpad), dtype=torch.float16, device=x_nchw.device)
    check(lib.ih_im2col3x3_nchw_f16(x_nchw.data_ptr(), out.data_ptr(), B, Cin, H, W, kpad, _stream()),
          "ih_im2col3x3_nchw_f16")
    return out


def im2col3x3_nchw_cat(x0: torch.Tensor, x1: torch.Tensor, kpad: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """im2col3x3_nchw of torch.cat([x0, x1], 1) without forming the concatenation: x0 [B, C0, H, W], x1 [B, C1, H, W]
    -> A [B*H*W, kpad] (conv_in of the 9-channel inpainting UNet: latents | mask | masked-image latents)."""
    lib = _lib.load()
    _req(x0, "x0")
    _req(x1, "x1")
    B, C0, H, W = x0.shape
    if x1.dim() != 4 or x1.shape[0] != B or tuple(x1.shape[2:]) != (H, W):
        raise IHError(f"im2col3x3_nchw_cat: x1 {tuple(x1.shape)} does not match x0 {tuple(x0.shape)}")
    if out is None:
        out = torch.empty((B * H * W, kpad), dtype=torch.float16, device=x0.device)
    check(lib.ih_im2col3x3_nchw_cat_f16(x0.data_ptr(), C0, x1.data_ptr(), x1.shape[1], out.data_ptr(), B, H, W, kpad,
                                        _stream()), "ih_im2col3x3_nchw_cat_f16")
    return out


def softmax_rows_masked_(x: torch.Tensor, valid_cols: int) -> torch.Tensor:
    """In-place softmax of a 2-D fp16 matrix (row stride arbitrary, cols % 8 == 0, <= 32768) over the first `valid_cols`
    columns of each row; the remaining (padding) columns become 0."""
    lib = _lib.load()
    _req(x, "x")
    if x.dim() != 2 or not 0 < valid_cols <= x.shape[1]:
        raise IHError("softmax_rows_masked_: 2-D matrix and 0 < valid_cols <= cols required")
    check(lib.ih_softmax_rows_masked_f16(x.data_ptr(), _rows(x, "x"), x.shape[0], x.shape[1], int(valid_cols), _stream()),
          "ih_softmax_rows_masked_f16")
    return x


def nhwc_to_nchw(x: torch.Tensor, C: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x NHWC [B, H, W, ldc] -> NCHW [B, C, H, W] taking channels [0, C)."""
    lib = _lib.load()
    _req(x, "x")
    B, H, W, ldc = x.shape
    if out is None:
        out = torch.empty((B, C, H, W), dtype=torch.float16, device=x.device)
    check(lib.ih_nhwc_to_nchw_f16(x.data_ptr(), ldc, out.data_ptr(), B, H * W, C, _stream()), "ih_nhwc_to_nchw_f16")
    return out


def euler_cfg_step(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, sigmas: torch.Tensor,
                   step: torch.Tensor, guidance: float) -> None:
    lib = _lib.load()
    _req(noise_pred, "noise_pred"); _req(latents, "latents"); _req(model_in, "model_in")
    _req(sigmas, "sigmas", torch.float32); _req(step, "step", torch.int32)
    n = latents.shape[0]
    per = latents.numel() // n
    check(lib.ih_euler_cfg_step(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(), sigmas.data_ptr(),
                                step.data_ptr(), float(guidance), per, n, _stream()), "ih_euler_cfg_step")


def euler_step(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, sigmas: torch.Tensor,
               step: torch.Tensor, guidance: float, *, use_cfg: bool = True, guidance_rescale: float = 0.0) -> None:
    """One scheduler transition with the reference's loop options: the default (CFG, no rescale) is the fused
    grid-stride kernel `ih_euler_cfg_step`; guidance_scale <= 1 and guidance_rescale > 0 (custom_pipelines.py:223,
    :352-354) run `ih_euler_step_ex` (one block per image, per-image std for the rescale)."""
    if use_cfg and not guidance_rescale:
        return euler_cfg_step(noise_pred, latents, model_in, sigmas, step, guidance)
    lib = _lib.load()
    _req(noise_pred, "noise_pred"); _req(latents, "latents"); _req(model_in, "model_in")
    _req(sigmas, "sigmas", torch.float32); _req(step, "step", torch.int32)
    n = latents.shape[0]
    per = latents.numel() // n
    want = (2 * n if use_cfg else n) * per
    if noise_pred.numel() != want or model_in.numel() != want:
        raise IHError(f"euler_step: noise_pred / model_in must hold {want} elements (use_cfg={use_cfg})")
    check(lib.ih_euler_step_ex(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(), sigmas.data_ptr(),
                               step.data_ptr(), float(guidance), float(guidance_rescale), per, n, int(use_cfg),
                               _stream()), "ih_euler_step_ex")


def euler_inpaint_step(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, sigmas: torch.Tensor,
                       step: torch.Tensor, guidance: float, image_latents: torch.Tensor, noise: torch.Tensor,
                       mask: torch.Tensor, blend_end: torch.Tensor, *, use_cfg: bool = True,
                       guidance_rescale: float = 0.0) -> None:
    """euler_step followed by the inpainting blend (ih_euler_inpaint_step): outside `mask` the latents are replaced by
    `image_latents` re-noised to the next sigma, or by the clean `image_latents` after the step that ends the loop at
    schedule index `blend_end` (device int32).  image_latents / noise [n,4,h,w] and mask [n,1,h,w], fp16."""
    lib = _lib.load()
    _req(noise_pred, "noise_pred"); _req(latents, "latents"); _req(model_in, "model_in")
    _req(sigmas, "sigmas", torch.float32); _req(step, "step", torch.int32)
    _req(image_latents, "image_latents"); _req(noise, "noise"); _req(mask, "mask"); _req(blend_end, "blend_end", torch.int32)
    n, c, h, w = latents.shape
    per = latents.numel() // n
    want = (2 * n if use_cfg else n) * per
    if noise_pred.numel() != want or model_in.numel() != want:
        raise IHError(f"euler_inpaint_step: noise_pred / model_in must hold {want} elements (use_cfg={use_cfg})")
    if (c != 4 or tuple(image_latents.shape) != (n, 4, h, w) or tuple(noise.shape) != (n, 4, h, w)
            or tuple(mask.shape) != (n, 1, h, w)
            or not all(t.is_contiguous() for t in (latents, image_latents, noise, mask))):
        raise IHError(f"euler_inpaint_step: contiguous latents / image_latents / noise [{n}, 4, {h}, {w}] and mask "
                      f"[{n}, 1, {h}, {w}] required")
    check(lib.ih_euler_inpaint_step(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(), sigmas.data_ptr(),
                                    step.data_ptr(), float(guidance), float(guidance_rescale), per, n, int(use_cfg),
                                    image_latents.data_ptr(), noise.data_ptr(), mask.data_ptr(), blend_end.data_ptr(),
                                    _stream()), "ih_euler_inpaint_step")


def dpm_solver_step(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, prev_x0: torch.Tensor,
                    coeffs: torch.Tensor, step: torch.Tensor, loop_begin: torch.Tensor, guidance: float, *,
                    use_cfg: bool = True, guidance_rescale: float = 0.0,
                    unipc: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> None:
    """One multistep-solver transition (ih_dpm_solver_step) with the loop options of euler_step.  loop_begin: device
    int32, the schedule index whose step has no history; coeffs is indexed by the device step counter.

    DPM-Solver++ 2M (`unipc` None): the guided prediction's data estimate x0 goes to `prev_x0` for the next step, the
    new latents to `latents` and, unscaled, to `model_in`; coeffs: fp32 [T, 8] (DPMSolverMultistepScheduler.coeffs).

    UniPC (`unipc` = (last_sample, prev_x0_2)): the corrector rewrites the latents from `last_sample` and the data
    predictions of the two previous steps (`prev_x0`, `prev_x0_2`), the history shifts, and the predictor writes the
    new latents to `latents` and, unscaled, to `model_in`; coeffs: fp32 [T, 16] (UniPCMultistepScheduler.coeffs).
    Its bit-exact kernel test is tests/test_unipc_gpu.py::test_unipc_step_kernel (the op census lists the DPM-Solver++
    test for this op)."""
    lib = _lib.load()
    _req(noise_pred, "noise_pred"); _req(latents, "latents"); _req(model_in, "model_in"); _req(prev_x0, "prev_x0")
    _req(coeffs, "coeffs", torch.float32); _req(step, "step", torch.int32); _req(loop_begin, "loop_begin", torch.int32)
    n = latents.shape[0]
    per = latents.numel() // n
    want = (2 * n if use_cfg else n) * per
    if noise_pred.numel() != want or model_in.numel() != want:
        raise IHError(f"dpm_solver_step: noise_pred / model_in must hold {want} elements (use_cfg={use_cfg})")
    hist = (prev_x0,)
    if unipc is not None:
        _req(unipc[0], "last_sample"); _req(unipc[1], "prev_x0_2")
        hist += tuple(unipc)
    if any(t.shape != latents.shape for t in hist) or not all(t.is_contiguous() for t in (latents,) + hist):
        raise IHError("dpm_solver_step: contiguous latents, prev_x0 (and last_sample, prev_x0_2) of one shape required")
    width = 8 if unipc is None else IH_UNIPC_COEFFS
    if coeffs.dim() != 2 or coeffs.shape[1] != width or not coeffs.is_contiguous():
        raise IHError(f"dpm_solver_step: coeffs must be a contiguous [T, {width}] table")
    solver, extra = ((IH_SOLVER_DPMPP_2M, (None, None)) if unipc is None
                     else (IH_SOLVER_UNIPC_BH2, (unipc[0].data_ptr(), unipc[1].data_ptr())))
    check(lib.ih_dpm_solver_step(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(), prev_x0.data_ptr(),
                                 coeffs.data_ptr(), step.data_ptr(), loop_begin.data_ptr(), float(guidance),
                                 float(guidance_rescale), per, n, int(use_cfg), _stream(), solver, *extra),
          "ih_dpm_solver_step")


def euler_ancestral_step(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, coeffs: torch.Tensor,
                         step_noise: torch.Tensor, step: torch.Tensor, guidance: float, *, use_cfg: bool = True,
                         guidance_rescale: float = 0.0,
                         inpaint: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]] = None) -> None:
    """One Euler Ancestral transition (ih_euler_ancestral_step) with the loop options of euler_step.  coeffs: fp32
    [T, 8] (EulerAncestralDiscreteScheduler.coeffs) and step_noise: fp16 [T, n, C, h, w] (the Gaussian noise of every
    step, drawn by the caller), both indexed by the device step counter.  `inpaint` = (image_latents, noise, mask,
    blend_end) adds the blend of euler_inpaint_step."""
    lib = _lib.load()
    _req(noise_pred, "noise_pred"); _req(latents, "latents"); _req(model_in, "model_in"); _req(step_noise, "step_noise")
    _req(coeffs, "coeffs", torch.float32); _req(step, "step", torch.int32)
    n, c, h, w = latents.shape
    per = latents.numel() // n
    want = (2 * n if use_cfg else n) * per
    if noise_pred.numel() != want or model_in.numel() != want:
        raise IHError(f"euler_ancestral_step: noise_pred / model_in must hold {want} elements (use_cfg={use_cfg})")
    if coeffs.dim() != 2 or coeffs.shape[1] != 8 or not coeffs.is_contiguous():
        raise IHError("euler_ancestral_step: coeffs must be a contiguous [T, 8] table")
    if (step_noise.dim() != 5 or tuple(step_noise.shape[1:]) != (n, c, h, w) or step_noise.shape[0] != coeffs.shape[0]
            or not (step_noise.is_contiguous() and latents.is_contiguous())):
        raise IHError(f"euler_ancestral_step: contiguous latents and step_noise [{coeffs.shape[0]}, {n}, {c}, {h}, {w}] "
                      "required")
    blend = (None, None, None, None)
    if inpaint is not None:
        image_latents, noise, mask, blend_end = inpaint
        _req(image_latents, "image_latents"); _req(noise, "noise"); _req(mask, "mask")
        _req(blend_end, "blend_end", torch.int32)
        if (c != 4 or tuple(image_latents.shape) != (n, 4, h, w) or tuple(noise.shape) != (n, 4, h, w)
                or tuple(mask.shape) != (n, 1, h, w)
                or not all(t.is_contiguous() for t in (image_latents, noise, mask))):
            raise IHError(f"euler_ancestral_step: contiguous image_latents / noise [{n}, 4, {h}, {w}] and mask "
                          f"[{n}, 1, {h}, {w}] required")
        blend = (image_latents.data_ptr(), noise.data_ptr(), mask.data_ptr(), blend_end.data_ptr())
    check(lib.ih_euler_ancestral_step(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(),
                                      coeffs.data_ptr(), step_noise.data_ptr(), step.data_ptr(), float(guidance),
                                      float(guidance_rescale), per, n, int(use_cfg), *blend, _stream()),
          "ih_euler_ancestral_step")


def euler_ancestral_scale_input(latents: torch.Tensor, model_in: torch.Tensor, coeffs: torch.Tensor,
                                step: torch.Tensor, duplicate: bool = True) -> None:
    """The first model input of an Euler Ancestral loop: latents * coeffs[step, 6] (the fp32 reciprocal of
    sqrt(sigma^2 + 1)), rounded to fp16 as ATen rounds diffusers' scale_model_input."""
    lib = _lib.load()
    _req(latents, "latents"); _req(model_in, "model_in"); _req(coeffs, "coeffs", torch.float32)
    _req(step, "step", torch.int32)
    if model_in.numel() != (2 if duplicate else 1) * latents.numel():
        raise IHError("euler_ancestral_scale_input: model_in must hold the CFG pair (duplicate=True) or one copy")
    if coeffs.dim() != 2 or coeffs.shape[1] != 8 or not coeffs.is_contiguous():
        raise IHError("euler_ancestral_scale_input: coeffs must be a contiguous [T, 8] table")
    check(lib.ih_euler_ancestral_scale_input(latents.data_ptr(), model_in.data_ptr(), coeffs.data_ptr(),
                                             step.data_ptr(), latents.numel(), int(duplicate), _stream()),
          "ih_euler_ancestral_scale_input")


def scale_model_input(latents: torch.Tensor, model_in: torch.Tensor, sigmas: torch.Tensor, step: torch.Tensor,
                      duplicate: bool = True) -> None:
    lib = _lib.load()
    _req(latents, "latents"); _req(model_in, "model_in")
    if model_in.numel() != (2 if duplicate else 1) * latents.numel():
        raise IHError("scale_model_input: model_in must hold the CFG pair (duplicate=True) or one copy of the latents")
    check(lib.ih_scale_model_input_ex(latents.data_ptr(), model_in.data_ptr(), sigmas.data_ptr(), step.data_ptr(),
                                      latents.numel(), int(duplicate), _stream()), "ih_scale_model_input_ex")


def conv3x3_small(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor] = None, *, stride: int = 1,
                  silu: bool = False, nchw: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 conv, pad 1, stride 1 or 2, for small channel counts (ih_conv3x3_small_f16, the ControlNet conditioning
    embedding): x NHWC [B, H, W, Cin] (or NCHW [B, Cin, H, W] with nchw=True); w_packed [Cout, 9*Cin] tap-major;
    -> NHWC [B, ceil(H/stride), ceil(W/stride), Cout], bias and SiLU fused."""
    lib = _lib.load()
    _req(x, "x"); _req(w_packed, "w")
    if nchw:
        B, Cin, H, W = x.shape
        sb, sc, sh, sw = x.stride()
    else:
        B, H, W, Cin = x.shape
        sb, sh, sw, sc = x.stride()
    Cout = w_packed.shape[0]
    if not w_packed.is_contiguous() or w_packed.shape[1] != 9 * Cin:
        raise IHError(f"conv3x3_small: w_packed must be contiguous [Cout, {9 * Cin}], got {tuple(w_packed.shape)}")
    if bias is not None:
        _req(bias, "bias")
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), dtype=torch.float16, device=x.device)
    elif tuple(out.shape) != (B, Ho, Wo, Cout) or not out.is_contiguous():
        raise IHError(f"conv3x3_small: out must be contiguous {(B, Ho, Wo, Cout)}")
    rc = lib.ih_conv3x3_small_f16(x.data_ptr(), sb, sh, sw, sc, w_packed.data_ptr(), _p(bias), out.data_ptr(), B, H, W,
                                  Cin, Cout, stride, int(silu), _stream())
    check(rc, "ih_conv3x3_small_f16")
    return out


def controlnet_add_residuals(skips, residuals, scale: torch.Tensor, skip_row0s) -> None:
    """ih_controlnet_add_residuals_f16: skips[k][rows r0 .. r0 + R) = fp16(skip + fp16(residuals[k] * scale[k])) in
    place, all k in one launch.  skips[k] / residuals[k] are contiguous fp16 with the channel count last (the residual
    has R rows); scale is a device float32 vector with one value per entry; skip_row0s[k] is r0."""
    lib = _lib.load()
    _req(scale, "scale", torch.float32)
    n = len(skips)
    if not (n == len(residuals) == len(skip_row0s)) or scale.numel() < n or not scale.is_contiguous():
        raise IHError(f"controlnet_add_residuals: {n} skips, {len(residuals)} residuals, {len(skip_row0s)} offsets "
                      f"and {scale.numel()} scales")
    table = (_lib.IhCnResidual * n)()
    for k, (s, r, r0) in enumerate(zip(skips, residuals, skip_row0s)):
        _req(s, f"skip[{k}]"); _req(r, f"residual[{k}]")
        C = s.shape[-1]
        rows = r.numel() // C
        if (not s.is_contiguous() or not r.is_contiguous() or r.shape[-1] != C or r0 < 0
                or r0 + rows > s.numel() // C):
            raise IHError(f"controlnet_add_residuals: entry {k}: skip {tuple(s.shape)} cannot take residual "
                          f"{tuple(r.shape)} at row {r0}")
        table[k] = _lib.IhCnResidual(s.data_ptr(), r.data_ptr(), rows, int(r0), C)
    check(lib.ih_controlnet_add_residuals_f16(table, n, scale.data_ptr(), _stream()), "ih_controlnet_add_residuals_f16")


def controlnet_add_residuals_multi(skips, residuals_per_net, scales_per_net, skip_row0s) -> None:
    """ih_controlnet_add_residuals_multi_f16: for every entry k, skips[k][rows r0 .. r0 + R) = fp16(skip + acc) in
    place with acc = fp16(r_0 * s_0[k]), then acc = fp16(acc + fp16(r_j * s_j[k])) for the nets j = 1 .. K-1 in order
    (diffusers' MultiControlNetModel sum, then the UNet's addition), all entries and nets in one launch.
    residuals_per_net[j][k] is net j's residual for skip k (contiguous fp16, R rows); scales_per_net[j] is net j's
    device float32 vector with one value per entry; skip_row0s[k] is r0."""
    lib = _lib.load()
    K = len(residuals_per_net)
    n = len(skips)
    if not 1 <= K <= _lib.IH_CN_MAX_NETS or len(scales_per_net) != K:
        raise IHError(f"controlnet_add_residuals_multi: {K} residual lists and {len(scales_per_net)} scale vectors "
                      f"(1 .. {_lib.IH_CN_MAX_NETS} nets)")
    if len(skip_row0s) != n or any(len(rs) != n for rs in residuals_per_net):
        raise IHError(f"controlnet_add_residuals_multi: {n} skips, {[len(rs) for rs in residuals_per_net]} residuals "
                      f"per net, {len(skip_row0s)} offsets")
    for j, sc in enumerate(scales_per_net):
        _req(sc, f"scale[{j}]", torch.float32)
        if sc.numel() < n or not sc.is_contiguous():
            raise IHError(f"controlnet_add_residuals_multi: net {j} has {sc.numel()} scales for {n} entries")
    table = (_lib.IhCnMultiResidual * n)()
    for k, (s, r0) in enumerate(zip(skips, skip_row0s)):
        _req(s, f"skip[{k}]")
        C = s.shape[-1]
        rows = residuals_per_net[0][k].numel() // C
        for j, rs in enumerate(residuals_per_net):
            r = rs[k]
            _req(r, f"residual[{j}][{k}]")
            if (not s.is_contiguous() or not r.is_contiguous() or r.shape[-1] != C or r.numel() != rows * C or r0 < 0
                    or r0 + rows > s.numel() // C):
                raise IHError(f"controlnet_add_residuals_multi: entry {k}: skip {tuple(s.shape)} cannot take net {j}'s "
                              f"residual {tuple(r.shape)} at row {r0}")
        table[k] = _lib.IhCnMultiResidual(s.data_ptr(), rows, int(r0), C,
                                          (ctypes.c_void_p * _lib.IH_CN_MAX_NETS)(
                                              *[rs[k].data_ptr() for rs in residuals_per_net]))
    scales = (ctypes.c_void_p * K)(*[sc.data_ptr() for sc in scales_per_net])
    check(lib.ih_controlnet_add_residuals_multi_f16(table, n, scales, K, _stream()),
          "ih_controlnet_add_residuals_multi_f16")
