"""Edge-case GPU parity tests of kernels that the model goldens reach at one shape only: the small CUDA-core kernels,
the layout / pointwise kernels, the GEMM epilogue matrix on every tile width, GroupNorm and LayerNorm statistics.

References are fp64 PyTorch.  Where a kernel documents its fp16 rounding points, a second reference rounds at exactly
those points and the kernel must match it to about one fp16 ulp; the exact fp64 reference then gets a looser bar.
Inputs of the CUDA-core kernels are quantised (few mantissa bits) so that their fp32 sums are exact in any order and the
rounded reference meets the same values at every rounding point.
"""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from census import stats_ratio
from fp16_ulps import close_ulps, ulp16
from imagharmony_b200 import _lib
from imagharmony_b200._lib import IHError
from test_kernels_gpu import check, ops, rnd  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# IH_GN_FUSED is read once per process; test_groupnorm_two_kernel_path re-runs the GroupNorm cases in a child with "0"
GN_TWO_KERNEL = os.environ.get("IH_GN_FUSED", "1")[:1] == "0"


def r16(t):
    """Round to fp16 and continue in fp64 (a rounding point of the kernel)."""
    return t.half().double()


def qrnd(*shape, step=0.125, scale=1.0, seed=0):
    """Gaussian values rounded to multiples of `step`: exactly representable in fp16, and their products and sums are
    exact in fp32 for the sizes used here."""
    g = torch.Generator(device="cpu").manual_seed(seed + 7 * sum(shape))
    return (torch.round(torch.randn(*shape, generator=g, dtype=torch.float64) * scale / step) * step).half().cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------------
# ih_attention_small_f16: scores = fp16(fp16(q k^T) / scale), softmax in fp32, p rounded to fp16, out = fp16(p v)
# ------------------------------------------------------------------------------------------------------------
def _attention_small_case(ops, B, H, Nq, Nk, dqk, dv, qk_scale, pad=0, seed=0):
    scale = math.sqrt(dqk)
    # strided views: every operand is a column slice of a wider buffer
    qb = qrnd(B * Nq, H * dqk + 2 * pad, scale=qk_scale, seed=seed)
    kb = qrnd(B * Nk, H * dqk + 2 * pad, scale=qk_scale, seed=seed + 1)
    vb = qrnd(B * Nk, H * dv + 2 * pad, step=1 / 64, seed=seed + 2)
    q, k, v = qb[:, pad:pad + H * dqk], kb[:, pad:pad + H * dqk], vb[:, pad:pad + H * dv]
    ob = torch.zeros(B * Nq, H * dv + 2 * pad, dtype=torch.float16, device="cuda")
    out = ops.attention_small(q, k, v, B, H, Nq, Nk, dqk, dv, scale, out=ob[:, pad:pad + H * dv])
    if pad:
        assert (ob[:, :pad] == 0).all() and (ob[:, pad + H * dv:] == 0).all(), "wrote outside the output view"
    qd = q.double().reshape(B, Nq, H, dqk).transpose(1, 2)
    kd = k.double().reshape(B, Nk, H, dqk).transpose(1, 2)
    vd = v.double().reshape(B, Nk, H, dv).transpose(1, 2)
    s = qd @ kd.transpose(-1, -2)                                  # exact: quantised inputs
    scale32 = torch.tensor(scale, dtype=torch.float32).item()      # the kernel divides by the fp32 value
    s16 = r16(r16(s) / scale32)
    e = torch.exp(s16 - s16.amax(-1, keepdim=True))
    p16 = r16(e / e.sum(-1, keepdim=True))
    rounded = r16(p16 @ vd)
    mag = p16 @ vd.abs()
    exact_p = (s / scale).softmax(-1)
    exact = exact_p @ vd
    flat = lambda t: t.transpose(1, 2).reshape(B * Nq, H * dv)   # noqa: E731
    what = f"attention_small B{B} H{H} {Nq}x{Nk} d{dqk}/{dv}"
    # slack: __expf and the fp32 sums can push a few p_j across an fp16 rounding boundary (one ulp of that p_j each),
    # and the fp32 PV sum is not exact
    flips = 2 * (ulp16(p16)[..., None] * vd.abs()[:, :, None]).amax(dim=-2)
    close_ulps(out, flat(rounded), what + " (rounding points)",
               slack=flat(flips + mag * math.sqrt(Nk) * 2.0 ** -23))
    # the exact result differs by the score rounding: each p_j moves by at most ulp16(max|s|) relatively, p and out
    # are rounded once more
    bar = (ulp16(s16.abs().amax(-1, keepdim=True)) + 2.0 ** -10) * (exact_p @ vd.abs()) + 1e-4
    err = (out.double().reshape(B, Nq, H, dv).transpose(1, 2) - exact).abs()
    assert (err <= bar).all(), f"{what} vs fp64: max err {err.max().item():.3e}"
    return s16


@pytest.mark.parametrize("B", [1, 3])
def test_attention_small_harmony_shape(ops, B):
    _attention_small_case(ops, B, 10, 8, 77, 32, 64, qk_scale=1.0)


@pytest.mark.parametrize("Nk", [1, 31, 32, 33, 1024])
def test_attention_small_key_tails(ops, Nk):
    _attention_small_case(ops, 1, 2, 8, Nk, 40, 64, qk_scale=1.0, seed=Nk)


def test_attention_small_strided_views(ops):
    _attention_small_case(ops, 2, 3, 4, 50, 24, 40, qk_scale=1.0, pad=16)


def test_attention_small_wide_score_spread(ops):
    s16 = _attention_small_case(ops, 2, 4, 8, 200, 32, 64, qk_scale=2.8, seed=5)
    assert s16.abs().max().item() >= 20.0, "scores must spread to about +-30"


def test_attention_small_rejects_ragged_warp_count(ops):
    q, k, v = rnd(3, 32), rnd(5, 32), rnd(5, 64)
    with pytest.raises(IHError):
        ops.attention_small(q, k, v, 1, 1, 3, 5, 32, 64, math.sqrt(32))


# ------------------------------------------------------------------------------------------------------------
# ih_conv3x3_small_f16: out = fp16(act(bias + sum x w)), fp32 accumulation
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,Cin,Cout,stride,nchw,bias,silu", [
    (1, 7, 9, 3, 16, 1, True, True, True),       # the control image (NCHW, 3 channels)
    (2, 7, 9, 3, 16, 2, True, False, False),     # odd H / W at stride 2: Ho = ceil(H / 2)
    (1, 1, 1, 16, 16, 1, False, True, True),
    (3, 1, 1, 16, 96, 2, False, False, True),
    (2, 65, 97, 16, 32, 1, False, True, True),   # 520 x 776 image / 8
    (1, 65, 97, 32, 32, 2, False, True, False),
    (1, 65, 97, 96, 256, 2, False, True, True),
    (2, 9, 7, 96, 96, 1, False, False, False),
    (1, 65, 97, 3, 16, 1, True, True, True),
    (2, 13, 11, 32, 256, 2, True, True, True),   # NCHW strides at a wider channel count
])
def test_conv3x3_small_edges(ops, B, H, W, Cin, Cout, stride, nchw, bias, silu):
    x_nchw = qrnd(B, Cin, H, W, seed=1)
    x = x_nchw if nchw else x_nchw.permute(0, 2, 3, 1).contiguous()
    w = qrnd(Cout, Cin, 3, 3, step=1 / 256, scale=0.25, seed=2)
    b = qrnd(Cout, scale=0.5, seed=3) if bias else None
    out = ops.conv3x3_small(x, ops.pack_conv3x3_weight(w), b, stride=stride, silu=silu, nchw=nchw)
    acc = F.conv2d(x_nchw.double(), w.double(), None if b is None else b.double(), stride=stride, padding=1)
    if silu:
        acc = F.silu(acc)
    ref = acc.permute(0, 2, 3, 1)
    assert out.shape == (B, (H + stride - 1) // stride, (W + stride - 1) // stride, Cout)
    close_ulps(out, r16(ref), f"conv3x3_small {B}x{H}x{W} {Cin}->{Cout} s{stride} nchw{nchw} bias{bias} silu{silu}")


# ------------------------------------------------------------------------------------------------------------
# ih_linear_small_f16: y = fp16(W x + b); act_out; fp16(y) * out_scale; fp16(.) + addend; fp16   (pointwise.cu)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [8, 264, 2816])
@pytest.mark.parametrize("M", [1, 7, 8, 9, 17, 64])
def test_linear_small_edges(ops, M, K):
    N = 328
    xb = qrnd(M, K + 16, scale=2.0, seed=M)
    x = xb[:, 8:8 + K]                                               # row stride K + 16
    w = qrnd(N, K, step=1 / 256, scale=K ** -0.5, seed=K)
    b = qrnd(N, step=1 / 64, seed=1)
    addb = qrnd(M, N + 24, step=1 / 64, seed=2)
    addend = addb[:, 16:16 + N]                                      # row stride N + 24
    for act_in, act_out, scale, use_add in [(False, False, 1.0, False), (True, False, 1.0, False),
                                            (False, True, 1.0, False), (True, True, 0.7, True),
                                            (False, False, 1.3, True)]:
        ob = torch.zeros(M, N + 16, dtype=torch.float16, device="cuda")
        out = ops.linear_small(x, w, b, act_in=act_in, act_out=act_out, out_scale=scale,
                               addend=addend if use_add else None, out=ob[:, 8:8 + N])
        assert (ob[:, :8] == 0).all() and (ob[:, 8 + N:] == 0).all()
        xe = x.double()
        if act_in:
            xe = r16(F.silu(xe))                                     # the SiLU output is an fp16 tensor
        acc = xe @ w.double().t() + b.double()
        s32 = torch.tensor(scale, dtype=torch.float32).item()       # the kernel multiplies by the fp32 value
        y, yx = r16(acc), acc
        if act_out:
            y, yx = F.silu(y), F.silu(yx)
        if scale != 1.0:
            y, yx = r16(y) * s32, yx * scale
        if use_add:
            y, yx = r16(y) + addend.double(), yx + addend.double()
        what = f"linear_small M{M} K{K} in{act_in} out{act_out} s{scale} add{use_add}"
        # fp32 products of fp16 SiLU outputs are not exact: allow for the accumulation order; and a SiLU (fp32 __expf)
        # can move an intermediate rounding by one ulp, which the scale carries and an addend may expose by cancellation
        slack = (xe.abs() @ w.double().abs().t()) * 2.0 ** -20
        if act_in or act_out:
            slack = slack + ulp16(r16(acc)) * abs(s32)
        close_ulps(out, r16(y), what + " (rounding points)", slack=slack)
        check(out, yx, what + " (fp64)", rtol=4e-3, atol=4e-3)


# ------------------------------------------------------------------------------------------------------------
# layout and pointwise kernels
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,period", [(4096, 4096), (16 * 1280, 1280), (3 * 257 * 8, 8), (77 * 2048, 2048)])
def test_add_bcast(ops, n, period):
    a, b = rnd(n, seed=1), rnd(period, seed=2)
    out = ops.add_bcast(a, b)
    ref = (a.float() + b.float().repeat(n // period)).half()       # one fp16 rounding of the fp32 sum
    assert torch.equal(out, ref)


@pytest.mark.parametrize("D", [8, 1280, 2048])
@pytest.mark.parametrize("n", [1, 257, 4096])
def test_mean_tokens(ops, n, D):
    x = qrnd(2, n, D, step=1 / 16, seed=n)
    out = ops.mean_tokens(x)
    # the fp32 sums are exact; the kernel multiplies by the fp32 reciprocal of n
    close_ulps(out, r16(x.double().mean(dim=1)), f"mean_tokens n{n} D{D}")


@pytest.mark.parametrize("C,ldc", [(1, 8), (4, 16), (4, 4), (3, 320)])
def test_nhwc_to_nchw(ops, C, ldc):
    x = rnd(3, 5, 7, ldc)
    out = ops.nhwc_to_nchw(x, C)
    assert torch.equal(out, x[..., :C].permute(0, 3, 1, 2).contiguous())


@pytest.mark.parametrize("C0,C1", [(8, 8), (8, 320), (1280, 8)])
def test_concat_channels(ops, C0, C1):
    x0, x1 = rnd(3, 5, 7, C0, seed=1), rnd(3, 5, 7, C1, seed=2)
    assert torch.equal(ops.concat_channels(x0, x1), torch.cat([x0, x1], -1))


@pytest.mark.parametrize("H,W,C", [(1, 1, 8), (3, 5, 16), (7, 9, 640), (33, 17, 8)])
def test_upsample2x_odd(ops, H, W, C):
    x = rnd(2, H, W, C)
    out = ops.upsample2x(x)
    assert torch.equal(out, x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))


def test_embed_tokens_clamps_ids(ops):
    vocab, T, C = 50, 7, 64
    tok, pos = rnd(vocab, C, seed=1), rnd(T + 3, C, seed=2)
    ids = torch.tensor([[0, 49, 50, 1000, -1, -77, 3], [5, 6, 7, 2 ** 31 - 1, -2 ** 31, 48, 1]], dtype=torch.int32,
                       device="cuda")
    out = ops.embed_tokens(ids, tok, pos)
    want = (tok[ids.long().clamp(0, vocab - 1)].float() + pos[:T].float()[None]).half().reshape(-1, C)
    assert torch.equal(out, want)


# ------------------------------------------------------------------------------------------------------------
# GEMM / conv epilogue matrix on every tile width
# ------------------------------------------------------------------------------------------------------------
TILES = [64, 128, 160, 192, 256]


@pytest.mark.parametrize("M", [333, 1000])
@pytest.mark.parametrize("tile_n", TILES)
def test_gemm_epilogue_matrix(ops, tile_n, M):
    """bias + rowbias (groups not dividing M) + residual + each activation, N clipped in the last tile, strided output
    and residual views.  ReLU acts after the residual and goes through ih_gemm_f16 itself (ops.linear takes no tile_n
    or rowbias with it); on the 64- and 160-column tiles also with `stats_out`, whose slots must sum the stored ReLU'd
    values."""
    lib = _lib.load()
    K, N = 320, 2 * tile_n + 40
    rpg = 100 if M == 333 else 300
    x, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    rb = rnd(-(-M // rpg), N + 8, seed=4)[:, 8:]
    resb = rnd(M, N + 24, seed=5)
    res = resb[:, 16:16 + N]
    base = x.double() @ w.double().t() + b.double() + rb.double()[torch.arange(M, device="cuda") // rpg]
    for act, fn in [("none", lambda t: t), ("silu", F.silu), ("gelu", F.gelu),
                    ("quick_gelu", lambda t: t * torch.sigmoid(1.702 * t))]:
        ob = torch.zeros(M, N + 16, dtype=torch.float16, device="cuda")
        out = ops.linear(x, w, b, rowbias=rb, rows_per_group=rpg, residual=res, out=ob[:, 8:8 + N], tile_n=tile_n,
                         silu=act == "silu", gelu=act == "gelu", quick_gelu=act == "quick_gelu")
        assert (ob[:, :8] == 0).all() and (ob[:, 8 + N:] == 0).all(), "wrote outside the output view"
        check(out, fn(base) + res.double(), f"gemm bn{tile_n} M{M} N{N} {act}")
    ob = torch.zeros(M, N + 16, dtype=torch.float16, device="cuda")
    rc = lib.ih_gemm_f16(x.data_ptr(), K, w.data_ptr(), b.data_ptr(), rb.data_ptr(), rpg, rb.stride(0), res.data_ptr(),
                         res.stride(0), ob[:, 8:].data_ptr(), ob.stride(0), M, N, K, ops.EPI_RELU, tile_n, stream())
    _lib.check(rc, "ih_gemm_f16 relu")
    assert (ob[:, :8] == 0).all() and (ob[:, 8 + N:] == 0).all(), "wrote outside the output view"
    relu = torch.relu(base + res.double())
    assert bool((relu == 0).float().mean() > 0.2), "the ReLU must clip a good share of the outputs"
    check(ob[:, 8:8 + N], relu, f"gemm bn{tile_n} M{M} N{N} relu")
    if tile_n in (64, 160):
        Ns = 640                                              # stats_out: N % 64 == 0, and N % 320 == 0 at 160 columns
        ws, bs, rs = rnd(Ns, K, scale=K ** -0.5, seed=6), rnd(Ns, seed=7), rnd(M, Ns, seed=8)
        rbs = rnd(-(-M // rpg), Ns + 8, seed=9)[:, 8:]
        stats = torch.full((Ns // 64, M, 2), float("nan"), dtype=torch.float32, device="cuda")
        out = torch.empty(M, Ns, dtype=torch.float16, device="cuda")
        rc = lib.ih_gemm_ln_f16(x.data_ptr(), K, ws.data_ptr(), bs.data_ptr(), rbs.data_ptr(), rpg, rbs.stride(0),
                                rs.data_ptr(), Ns, out.data_ptr(), Ns, M, Ns, K, ops.EPI_RELU, tile_n, None, 0, 0.0,
                                stats.data_ptr(), stream())
        _lib.check(rc, "ih_gemm_ln_f16 relu stats_out")
        want = (x.double() @ ws.double().t() + bs.double() + rbs.double()[torch.arange(M, device="cuda") // rpg]
                + rs.double())
        check(out, torch.relu(want), f"gemm bn{tile_n} M{M} N{Ns} relu stats_out")
        assert stats_ratio(stats, out) <= 1.0, f"bn{tile_n} M{M}: slot sums are not those of the stored ReLU'd values"


def test_gemm_alpha_with_residual_and_gelu(ops):
    M, N, K = 1000, 360, 512
    x, w, b, res = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)
    alpha = 0.37
    out = ops.linear(x, w, b, residual=res, gelu=True, alpha=alpha)
    check(out, F.gelu(alpha * (x.double() @ w.double().t()) + b.double()) + res.double(), "gemm alpha gelu residual")


@pytest.mark.parametrize("H,W", [(13, 19), (20, 28)])
@pytest.mark.parametrize("tile_n", TILES)
def test_conv3x3_rowbias_every_tile(ops, tile_n, H, W):
    B, Cin, Cout = 3, 64, 360
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b, temb, res = rnd(Cout, seed=3), rnd(B, Cout + 64, seed=4), rnd(B, H, W, Cout, seed=5)
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, rowbias=temb[:, 64:], residual=res, tile_n=tile_n)
    ref = (F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
           + temb[:, 64:].double()[:, None, None, :] + res.double())
    check(out, ref, f"conv3x3 rowbias bn{tile_n} {B}x{H}x{W}")


def test_conv2d_scaled_stride2_residual(ops):
    """alpha * conv(x) + bias + residual at stride 2 and four output widths, and with IH_EPI_RELU relu of that sum."""
    B, H, W, Cin = 2, 30, 46, 128
    x = rnd(B, H, W, Cin, seed=1)
    for Cout in (192, 128, 320, 360):
        w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
        b, res = rnd(Cout, seed=3), rnd(B, H // 2, W // 2, Cout, seed=4)
        conv = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None, stride=2, padding=1).permute(0, 2, 3, 1)
        want = 0.125 * conv + b.double() + res.double()
        assert bool((want < 0).double().mean() > 0.2), "the ReLU must clip a good share of the outputs"
        for relu in (False, True):
            out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, stride=2, residual=res, alpha=0.125, relu=relu)
            check(out, torch.relu(want) if relu else want,
                  f"conv2d_scaled s2 + residual Cout {Cout}{' relu' if relu else ''}")


def _nonfinite_like_relu(out, ref, what):
    """ref: the fp64 reference before the ReLU.  out's NaN, +inf and -inf elements are exactly those of torch.relu(ref)
    (NaN and +inf pass, -inf becomes 0), and its other elements are within check's bar."""
    want = torch.relu(ref)
    for kind in (torch.isnan, torch.isposinf, torch.isneginf):
        assert torch.equal(kind(out), kind(want)), f"{what}: {kind.__name__} elements differ"
    fin = torch.isfinite(want)
    assert bool((~fin).any()) and bool(fin.any())
    check(out[fin], want[fin], what)


def test_relu_epilogue_propagates_nan_and_inf(ops):
    """IH_EPI_RELU keeps NaN as torch.relu does: NaN rows of the GEMM's A, a NaN input pixel of the conv at a
    spatial-tile corner, an image border and the batch boundary (its NaN footprint is exactly the 3x3 neighbourhood
    F.conv2d gives), and NaN / +inf / -inf in the residual."""
    from test_unet_census_gpu import conv_tile
    nan, inf = float("nan"), float("inf")
    # GEMM: NaN rows at both sides of the 128-row tile boundary and in the last row; non-finite residual elements
    M, N, K = 300, 360, 320
    x, w, b, res = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)
    x[[0, 127, 128, 299]] = nan
    x[5, 17] = nan
    res[40, 7], res[200, 100], res[250, 359], res[251, 0] = nan, inf, -inf, -inf
    for alpha in (1.0, 0.5):
        out = ops.linear(x, w, b, residual=res, alpha=alpha, relu=True)
        ref = alpha * (x.double() @ w.double().t()) + b.double() + res.double()
        _nonfinite_like_relu(out, ref, f"gemm relu alpha {alpha}")
    # conv: 24 x 40 outputs run on 16 x 8 spatial tiles; (7, 15) is the bottom-right corner of the first tile
    B, H, W, C = 2, 24, 40, 64
    assert conv_tile(H, W) == (16, 8)
    xc = rnd(B, H, W, C, seed=5)
    # a tile corner, the top border, image 0's last pixel (next to image 1's first in memory), image 1's left border
    px = [(0, 7, 15), (0, 0, 20), (0, H - 1, W - 1), (1, 12, 0)]
    for i, y, xx in px:
        xc[i, y, xx, (7 * y + xx) % C] = nan
    wc = rnd(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=6)
    bc, rc = rnd(C, seed=7), rnd(B, H, W, C, seed=8)
    rc[1, 3, 30, 5], rc[1, 20, 2, 60], rc[0, 15, 33, 0] = nan, inf, -inf
    for stride in (1, 2):
        r = rc if stride == 1 else rnd(B, H // 2, W // 2, C, seed=9)
        out = ops.conv3x3(xc, ops.pack_conv3x3_weight(wc), bc, residual=r, stride=stride, relu=True)
        # in fp64 on the host: every output reads exactly its 3 x 3 window there
        xn = xc.double().cpu().permute(0, 3, 1, 2)
        conv = F.conv2d(xn, wc.double().cpu(), bc.double().cpu(), stride=stride, padding=1).permute(0, 2, 3, 1)
        window = F.max_pool2d(torch.isnan(xn).any(1, keepdim=True).double(), 3, stride, 1).bool().permute(0, 2, 3, 1)
        assert torch.equal(torch.isnan(conv), window.expand_as(conv)), "fp64 reference: NaN beyond the 3x3 windows"
        _nonfinite_like_relu(out, (conv + r.double().cpu()).cuda(), f"conv relu s{stride}")


# ------------------------------------------------------------------------------------------------------------
# the attention entry without a workspace, and the first-step input scaling
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Nq,Nk,n_ip", [(256, 81, 4), (300, 300, 0)])
def test_attention_ws_f16_without_workspace(ops, Nq, Nk, n_ip):
    """ih_attention_ws_f16 with workspace == NULL processes every query tile whole, as ops.attention(kv_split=False)."""
    lib = _lib.load()
    B, H = 2, 4
    q, k, v = rnd(B * Nq, H * 64), rnd(B * Nk, H * 64, seed=1), rnd(B * Nk, H * 64, seed=2)
    out = torch.empty(B * Nq, H * 64, dtype=torch.float16, device="cuda")
    rc = lib.ih_attention_ws_f16(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                 out.data_ptr(), out.stride(0), B, H, Nq, Nk, n_ip, 0.6, None, 0, stream())
    _lib.check(rc, "ih_attention_ws_f16")
    assert torch.equal(out, ops.attention(q, k, v, B, H, Nq, Nk, n_ip=n_ip, ip_scale=0.6, kv_split=False))
    nt = Nk - n_ip
    qd = q.double().reshape(B, Nq, H, 64).transpose(1, 2)
    kd = k.double().reshape(B, Nk, H, 64).transpose(1, 2)
    vd = v.double().reshape(B, Nk, H, 64).transpose(1, 2)
    ref = (qd @ kd[:, :, :nt].transpose(-1, -2) / 8).softmax(-1) @ vd[:, :, :nt]
    if n_ip:
        ref = ref + 0.6 * ((qd @ kd[:, :, nt:].transpose(-1, -2) / 8).softmax(-1) @ vd[:, :, nt:])
    check(out, ref.transpose(1, 2).reshape(B * Nq, H * 64), f"ih_attention_ws_f16 no workspace {Nq}x{Nk} ip{n_ip}")


def test_scale_model_input_entry(ops):
    """ih_scale_model_input_ex with the CFG duplicate: model_in = cat([x, x]) / sqrt(sigma[*step]^2 + 1)."""
    lat = rnd(3, 4, 24, 40) * 7
    sig = torch.tensor([14.6, 9.1, 0.03], device="cuda")
    step = torch.tensor([1], dtype=torch.int32, device="cuda")
    a = torch.empty(6, 4, 24, 40, dtype=torch.float16, device="cuda")
    ops.scale_model_input(lat, a, sig, step)
    mi = r16(lat.double() / math.sqrt(sig[1].item() ** 2 + 1))
    close_ulps(a, torch.cat([mi, mi]), "ih_scale_model_input_ex")
    assert int(step.item()) == 1, "the input scaling must not advance the step counter"


# ------------------------------------------------------------------------------------------------------------
# GroupNorm
# ------------------------------------------------------------------------------------------------------------
def gn_ref(x0, x1, gamma, beta, groups, eps, silu):
    x = x0 if x1 is None else torch.cat([x0, x1], -1)
    y = F.group_norm(x.double().permute(0, 3, 1, 2), groups, gamma.double(), beta.double(), eps)
    return (F.silu(y) if silu else y).permute(0, 2, 3, 1)


def gn_run(ops, x0, gamma, beta, **kw):
    """ops.groupnorm, asserting the launch shape: one fused launch, or statistics + apply with IH_GN_FUSED=0."""
    n0 = ops.launch_count()
    out = ops.groupnorm(x0, gamma, beta, **kw)
    assert ops.launch_count() - n0 == (2 if GN_TWO_KERNEL else 1)
    return out


def gn_params(C, seed=0):
    return (rnd(C, seed=seed) * 0.5 + 1).half(), rnd(C, seed=seed + 1) * 0.5


@pytest.mark.parametrize("C,groups,B,HW", [
    (320, 8, 1, 64), (320, 16, 3, 7), (640, 64, 8, 256), (1280, 32, 16, 64),
    (320, 160, 3, 1024),       # 2*groups > threads per block (240)
    (1280, 160, 1, 256),       # 160 threads for 320 values
    (1280, 160, 16, 64),
    (2048, 256, 2, 64),
    (1280, 640, 2, 64),        # C > 1024: the most groups the statistics buffer holds
    (1024, 1024, 1, 64),       # one channel per group
    (4096, 32, 1, 16),         # the largest C
])
def test_groupnorm_group_counts(ops, C, groups, B, HW):
    x = (rnd(B, HW, 1, C, seed=groups) * 1.5 + 0.3).half()
    g, b = gn_params(C)
    out = gn_run(ops, x, g, b, groups=groups, eps=1e-5, silu=True)
    check(out, gn_ref(x, None, g, b, groups, 1e-5, True), f"groupnorm C{C} g{groups} B{B} HW{HW}", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("C,B,HW", [
    (320, 16, 1), (1280, 1, 1), (1280, 8, 7),
    (320, 3, 23), (640, 8, 11), (1280, 2, 3), (2560, 3, 3),   # HW = 4R - 1: one block per image, a ragged row lane
])
def test_groupnorm_spatial_edges(ops, C, B, HW):
    x = rnd(B, HW, 1, C, seed=HW) * 2
    g, b = gn_params(C)
    out = gn_run(ops, x, g, b, eps=1e-5)
    check(out, gn_ref(x, None, g, b, 32, 1e-5, False), f"groupnorm C{C} B{B} HW{HW}", rtol=2e-3, atol=2e-3)


def test_groupnorm_vae_full_resolution(ops):
    """The VAE decoder's last level at 1024^2 (C=128, one image): 2^-7-scaled stream with eps = 1e-6 * s^2."""
    s = 2.0 ** -7
    x = (rnd(1, 1024, 1024, 128, seed=9) * (3 * s) + s).half()
    g, b = gn_params(128)
    out = gn_run(ops, x, g, b, eps=1e-6 * s * s, silu=True)
    check(out, gn_ref(x, None, g, b, 32, 1e-6 * s * s, True), "groupnorm VAE 1024^2", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("C0,C1,HW", [(1280, 1280, 1024), (1280, 640, 1024), (640, 640, 4096), (640, 320, 4096),
                                      (320, 320, 4096)])
def test_groupnorm_up_block_concat(ops, C0, C1, HW):
    """Every channel concat of the SDXL up-blocks (2560, 1920, 1280, 960, 640 channels)."""
    x0, x1 = rnd(2, HW, 1, C0, seed=1), rnd(2, HW, 1, C1, seed=2) * 3 - 0.5
    g, b = gn_params(C0 + C1)
    out = gn_run(ops, x0, g, b, x1=x1, silu=True)
    check(out, gn_ref(x0, x1, g, b, 32, 1e-5, True), f"groupnorm concat {C0}+{C1}", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("ratio", [8, 64])
@pytest.mark.parametrize("C,groups,B,HW", [(320, 32, 2, 4096), (1280, 32, 2, 1024), (640, 64, 8, 256),
                                           (1280, 160, 1, 1024)])
def test_groupnorm_large_group_means(ops, C, groups, B, HW, ratio):
    """Per-(image, group) offsets up to `ratio` standard deviations: E[x^2] - mean^2 from fp32 partial sums."""
    gen = torch.Generator(device="cpu").manual_seed(C + groups + ratio)
    std = torch.rand(B, 1, 1, groups, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    sign = torch.randint(0, 2, (B, 1, 1, groups), generator=gen).double() * 2 - 1
    mean = sign * std * ratio * (0.5 + 0.5 * torch.rand(B, 1, 1, groups, generator=gen, dtype=torch.float64))
    z = torch.randn(B, HW, 1, C, generator=gen, dtype=torch.float64)
    x = (mean.repeat_interleave(C // groups, -1) + std.repeat_interleave(C // groups, -1) * z).half().cuda()
    g, b = gn_params(C)
    out = gn_run(ops, x, g, b, groups=groups, eps=1e-5)
    check(out, gn_ref(x, None, g, b, groups, 1e-5, False), f"groupnorm C{C} g{groups} |mean|/std<={ratio}",
          rtol=2e-3, atol=2e-3)


def test_groupnorm_workspace_reuse_and_graph_replay(ops):
    """Calls with different (B, groups) share one workspace; captured in one CUDA graph and replayed, every output is
    bit-identical to the eager run, and the ticket / ready / departure flags are back at zero after each run."""
    lib = _lib.load()
    calls = [(2, 32, 1280, 64), (8, 32, 320, 256), (1, 160, 1280, 64), (3, 16, 640, 100), (16, 32, 640, 16),
             (2, 32, 1280, 64)]
    need = max(int(lib.ih_groupnorm_workspace_bytes(B, gr)) for B, gr, _, _ in calls)
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    sync_bytes = 3 * 1024 * 4          # the uint32 flags at the start of the workspace (norm.cu GN_SYNC_WORDS)
    args = []
    for i, (B, gr, C, HW) in enumerate(calls):
        x = rnd(B, HW, 1, C, seed=10 + i) * (1 + i)
        g, b = gn_params(C, seed=i)
        args.append((x, g, b, gr, torch.empty_like(x)))

    def run_all():
        for x, g, b, gr, o in args:
            ops.groupnorm(x, g, b, groups=gr, silu=True, out=o, ws=ws)

    run_all()
    torch.cuda.synchronize()
    eager = [o.clone() for *_, o in args]
    for (x, g, b, gr, _), e in zip(args, eager):
        check(e, gn_ref(x, None, g, b, gr, 1e-5, True), f"groupnorm shared ws g{gr}", rtol=2e-3, atol=2e-3)
    assert (ws[:sync_bytes] == 0).all(), "flags not reset after the eager run"
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run_all()
    for rep in range(3):
        for *_, o in args:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for i, ((*_, o), e) in enumerate(zip(args, eager)):
            assert torch.equal(o, e), f"replay {rep}, call {i}: differs from the eager run"
        assert (ws[:sync_bytes] == 0).all(), f"flags not reset after replay {rep}"


@pytest.mark.skipif(GN_TWO_KERNEL, reason="this process already runs the two-kernel path")
def test_groupnorm_two_kernel_path():
    """The GroupNorm cases once more with IH_GN_FUSED=0 (statistics kernel + apply kernel); the flag is read once per
    process, so they run in a child process."""
    env = dict(os.environ, IH_GN_FUSED="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.abspath(__file__), "-k", "groupnorm and not two_kernel"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-2000:]


# ------------------------------------------------------------------------------------------------------------
# LayerNorm and the LayerNorm fold
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [100, 300])
@pytest.mark.parametrize("rows", [1, 3, 2049])
@pytest.mark.parametrize("C", [8, 264, 5120, 8192])
def test_layernorm_large_mean(ops, C, rows, offset):
    """Rows whose mean is `offset` standard deviations: the explicit kernel centres before squaring (two passes)."""
    x = (rnd(rows, C, seed=C) + offset).half()
    g, b = gn_params(C)
    out = ops.layernorm(x, g, b, 1e-5)
    check(out, F.layer_norm(x.double(), (C,), g.double(), b.double(), 1e-5), f"layernorm {rows}x{C} +{offset}",
          rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("ratio", [
    1, 4, 32,
    pytest.param(256, marks=pytest.mark.xfail(strict=True, reason="the fold's var = E[x^2] - mean^2 from fp32 slot "
                                                                  "sums cancels when |mean|/std is in the hundreds")),
])
def test_layernorm_fold_accuracy_envelope(ops, ratio):
    """test_gemm_layernorm_fold's criteria on rows offset + N(0, 1): the fold stays within the accuracy class of the
    unfused LayerNorm -> GEMM pipeline while |mean| / std is moderate: the folded weight's fp16 rows sum to zero
    (ops.fold_layernorm), so what is left is the consumer's cancellation in var = E[x^2] - mean^2."""
    M, K, N = 1024, 1280, 1280
    a = rnd(M, K, seed=41)
    wp = rnd(K, K, scale=K ** -0.5, seed=42)
    res = (ratio + 0.25 * rnd(M, 1, seed=43).float()).half().expand(M, K).contiguous()
    stats = torch.full(((K + 63) // 64, M, 2), float("nan"), dtype=torch.float32, device="cuda")
    h = ops.linear(a, wp, residual=res, stats_out=stats)
    hd = h.double()
    print(f"[ln_fold envelope] |mean|/std = {(hd.mean(1).abs() / hd.std(1)).median().item():.1f}")
    gamma = (1 + 0.2 * rnd(K, seed=45).float()).half()
    beta = (0.1 * rnd(K, seed=46).float()).half()
    w, b = rnd(N, K, scale=K ** -0.5, seed=47), rnd(N, scale=0.25, seed=48)
    w_c, c = ops.fold_layernorm(w, b, gamma, beta)
    out = ops.linear(h, w_c, c, ln=(stats, 1e-5))
    exact = F.layer_norm(hd, (K,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()
    unfused = ops.linear(ops.layernorm(h, gamma, beta, 1e-5), w, b)
    e_fold, e_unf = (out.double() - exact).abs(), (unfused.double() - exact).abs()
    rms_fold, rms_unf = e_fold.pow(2).mean().sqrt().item(), e_unf.pow(2).mean().sqrt().item()
    print(f"[ln_fold envelope ratio {ratio}] rms err fold {rms_fold:.3e} unfused {rms_unf:.3e}; "
          f"max fold {e_fold.max().item():.3e} unfused {e_unf.max().item():.3e}")
    assert torch.isfinite(out).all()
    assert rms_fold <= 1.5 * rms_unf + 1e-6, (rms_fold, rms_unf)
    assert e_fold.max().item() <= 2.0 * e_unf.max().item() + 1e-3
