"""GPU tests of the 128x160 tile of gemm_f16_kernel: SDXL's 320 * 2^k channel widths split into whole 160-column tiles.
The last 64-column staging slab of such a tile is only 32 columns wide; it must store exactly those columns (the next
tile owns the ones after it), and row statistics of a pair of tiles must cover its 5 slots exactly once."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

RTOL = ATOL = 1e-3


@pytest.fixture(scope="module")
def ops():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from imagharmony_b200 import ops as _ops
    return _ops


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def check(out, ref, what, rtol=RTOL, atol=ATOL):
    out, ref = out.float(), ref.float()
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs()
    tol = atol + rtol * ref.abs() + ref.abs() * 2.0 ** -11     # one fp16 rounding of the fp32 reference
    frac = (err > tol).float().mean().item()
    print(f"[{what}] max_abs_err={err.max().item():.3e} frac_out_of_tol={frac:.2e}")
    assert frac == 0.0, f"{what}: {frac:.3e} of elements out of tolerance, max err {err.max().item():.3e}"


@pytest.mark.parametrize("M,N,K", [
    (2048, 1280, 1280),    # level-2 to_q / to_out / proj
    (2048, 1280, 5120),    # level-2 FF-out
    (8192, 640, 640),      # level-1 to_q / to_out / proj
    (8192, 640, 2560),     # level-1 FF-out
    (2048, 3840, 1280),    # q|k|v
    (1000, 1280, 640),     # ragged M
    (154, 640, 2048),
    (1000, 200, 320),      # N not a multiple of 160: the second tile has 40 columns
    (300, 72, 200),        # N below one slab, K not a multiple of 64
    (512, 480, 640),       # N = 3 tiles: an odd last tile
])
def test_gemm_bn160_plain(ops, M, N, K):
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    out = ops.linear(x, w, tile_n=160)
    check(out, x.float() @ w.float().t(), f"gemm {M}x{N}x{K} bn160")
    # the k-order of the accumulation does not depend on the tile width
    assert torch.equal(out, ops.linear(x, w, tile_n=192))


def test_gemm_bn160_epilogues(ops):
    M, N, K = 2048, 1280, 640
    x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N)
    res = rnd(M, N, seed=3)
    rb = rnd(2, N, seed=5)
    base = x.float() @ w.float().t()
    check(ops.linear(x, w, b, tile_n=160), base + b.float(), "bias")
    check(ops.linear(x, w, b, residual=res, tile_n=160), base + b.float() + res.float(), "bias+residual")
    ref = base + b.float() + rb.float().repeat_interleave(M // 2, dim=0)
    check(ops.linear(x, w, b, rowbias=rb, rows_per_group=M // 2, tile_n=160), ref, "bias+rowbias")
    check(ops.linear(x, w, b, silu=True, tile_n=160), F.silu(base + b.float()), "bias+silu")
    check(ops.linear(x, w, b, gelu=True, tile_n=160), F.gelu(base + b.float()), "bias+gelu")
    # alpha has no tile argument: at M = 2048, N = 1280 the library's choice is the 160-column tile
    check(ops.linear(x, w, b, residual=res, alpha=0.25), 0.25 * base + b.float() + res.float(), "alpha+bias+residual")


@pytest.mark.parametrize("N", [1280, 200])
def test_gemm_bn160_strided_guard(ops, N):
    """Output and residual are column windows of wider buffers: the columns on both sides must stay untouched."""
    M, K, pad = 1000, 640, 40
    x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N)
    rbuf = rnd(M, N + 2 * pad, seed=9)
    res = rbuf[:, pad:pad + N]
    sentinel = 7.0
    obuf = torch.full((M, N + 2 * pad), sentinel, dtype=torch.float16, device="cuda")
    ops.linear(x, w, b, residual=res, out=obuf[:, pad:pad + N], tile_n=160)
    check(obuf[:, pad:pad + N], x.float() @ w.float().t() + b.float() + res.float(), f"strided N{N}")
    assert (obuf[:, :pad] == sentinel).all() and (obuf[:, pad + N:] == sentinel).all()


@pytest.mark.parametrize("M,N", [(2048, 1280), (8192, 640), (1000, 1280)])
def test_gemm_bn160_layernorm_fold(ops, M, N):
    """Producer with 160-column tiles: every statistics slot is written once and the slot sums are the rows' sums; the
    consumer's folded LayerNorm matches the explicit LayerNorm -> GEMM pipeline."""
    K = N
    a = rnd(M, K, seed=31)
    wp, bp = rnd(K, K, scale=K ** -0.5, seed=32), rnd(K, seed=33)
    res = rnd(M, K, seed=34) * 2 + 0.5
    stats = torch.full(((K + 63) // 64, M, 2), float("nan"), dtype=torch.float32, device="cuda")
    h = ops.linear(a, wp, bp, residual=res, stats_out=stats, tile_n=160)
    assert torch.isfinite(stats).all()
    hf = h.float()
    s = stats.sum(dim=0)
    torch.testing.assert_close(s[:, 0], hf.sum(dim=1), rtol=1e-5, atol=1e-3)
    torch.testing.assert_close(s[:, 1], (hf * hf).sum(dim=1), rtol=1e-5, atol=1e-3)
    assert torch.equal(h, ops.linear(a, wp, bp, residual=res, tile_n=192))

    gamma = (1 + 0.2 * rnd(K, seed=35).float()).half()
    beta = (0.1 * rnd(K, seed=36).float()).half()
    w, b = rnd(N, K, scale=K ** -0.5, seed=37), rnd(N, scale=0.25, seed=38)
    w_c, c = ops.fold_layernorm(w, b, gamma, beta)
    out = ops.linear(h, w_c, c, ln=(stats, 1e-5), tile_n=160)
    exact = (F.layer_norm(h.double(), (K,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()).float()
    unfused = ops.linear(ops.layernorm(h, gamma, beta, 1e-5), w, b).float()
    e_fold, e_unf = (out.float() - exact).abs(), (unfused - exact).abs()
    assert torch.isfinite(out).all()
    assert e_fold.pow(2).mean().sqrt().item() <= 1.5 * e_unf.pow(2).mean().sqrt().item() + 1e-6
    assert e_fold.max().item() <= 2.0 * e_unf.max().item() + 1e-3
    check(out, exact, f"ln_fold M{M} N{N}", rtol=2e-3, atol=2e-3)


def test_gemm_bn160_stats_need_whole_tile_pairs(ops):
    from imagharmony_b200._lib import IHError
    M, N, K = 256, 1024, 320                              # 1024 = 6.4 tiles: the last pair is incomplete
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    stats = torch.full(((N + 63) // 64, M, 2), float("nan"), dtype=torch.float32, device="cuda")
    with pytest.raises(IHError):
        ops.linear(x, w, stats_out=stats, tile_n=160)
    h = ops.linear(x, w, stats_out=stats)                 # the library's choice avoids the 160-column tile
    assert torch.isfinite(stats).all()
    torch.testing.assert_close(stats.sum(dim=0)[:, 0], h.float().sum(dim=1), rtol=1e-5, atol=1e-3)


def conv_ref(x, w_packed, bias, stride=1, pad_br=False):
    Cout, Cin = w_packed.shape[0], x.shape[-1]
    w4 = w_packed[:, :9 * Cin].float().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    xn = x.float().permute(0, 3, 1, 2)
    if pad_br:
        y = F.conv2d(F.pad(xn, (0, 1, 0, 1)), w4, bias.float(), stride=2)
    else:
        y = F.conv2d(xn, w4, bias.float(), stride=stride, padding=1)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("H,C", [(32, 1280), (64, 640), (128, 320)])
@pytest.mark.parametrize("stride", [1, 2])
def test_conv_bn160(ops, H, C, stride):
    B = 2
    x, w, b = rnd(B, H, H, C), rnd(C, 9 * C, scale=(9 * C) ** -0.5), rnd(C)
    out = ops.conv3x3(x, w, b, stride=stride, tile_n=160)
    check(out, conv_ref(x, w, b, stride=stride), f"conv {H}^2 C{C} s{stride} bn160", rtol=2e-3, atol=2e-3)
    assert torch.equal(out, ops.conv3x3(x, w, b, stride=stride, tile_n=192))
    if stride == 1:
        res = rnd(B, H, H, C, seed=4)
        out = ops.conv3x3(x, w, b, residual=res, tile_n=160)
        check(out, conv_ref(x, w, b) + res.float(), f"conv+res {H}^2 C{C} bn160", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("H,C", [(64, 640), (32, 1280)])
def test_conv_down_bn160(ops, H, C):
    """Bottom/right-padded stride-2 conv (VAE encoder Downsample2D), with the output scale."""
    B = 2
    x, w, b = rnd(B, H, H, C), rnd(C, 9 * C, scale=(9 * C) ** -0.5), rnd(C)
    out = ops.conv3x3_down(x, w, b, tile_n=160, alpha=0.5)
    check(out, 0.5 * conv_ref(x, w, b * 2, pad_br=True), f"conv_down {H}^2 C{C} bn160", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("H,C,two", [(32, 1280, False), (32, 1280, True), (64, 640, True)])
def test_conv_shortcut_bn160(ops, H, C, two):
    """Fused 1x1 shortcut over one or two sources; the shortcut call has no tile argument, and at these shapes
    (M = 2048, N = 1280 and M = 8192, N = 640) the library's choice is the 160-column tile."""
    B = 2
    x = rnd(B, H, H, C)
    s0 = rnd(B, H, H, C, seed=11)
    s1 = rnd(B, H, H, C // 2, seed=12) if two else None
    csc = C + (C // 2 if two else 0)
    w, b = rnd(C, 9 * C + csc, scale=(9 * C + csc) ** -0.5), rnd(C)
    out = ops.conv3x3(x, w, b, shortcut=(s0, s1))
    src = torch.cat([s0, s1], dim=-1) if two else s0
    ref = conv_ref(x, w, b) + src.float() @ w[:, 9 * C:].float().t()
    check(out, ref, f"conv+shortcut {H}^2 C{C} two={two}", rtol=2e-3, atol=2e-3)
