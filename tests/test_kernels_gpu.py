"""GPU parity tests of the core C-ABI kernels (GEMM / conv, attention, norms, the Euler step and a few small kernels)
against a plain PyTorch fp32 reference of the same op (same fp16-rounded inputs). Tolerance: rtol = atol = 1e-3 on fp16
outputs unless a test states otherwise (BASELINE.json north_star). All calls go through imagharmony_b200.ops -> ctypes
-> libimagharmony_sm90.so. The edge cases of the shared kernels live in test_kernel_edges_gpu.py, the feature kernels
in their features' *_gpu.py files; test_kernel_coverage_cpu.py maps every entry point of include/ih_api.h to the tests
that call it directly.
"""
import math

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
    out = out.float()
    ref = ref.float()
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    # the reference is fp32; the kernel output is fp16 -> allow one fp16 rounding of the reference as well
    err = (out - ref).abs()
    tol = atol + rtol * ref.abs() + ref.abs() * 2.0 ** -11
    bad = (err > tol)
    frac = bad.float().mean().item()
    print(f"[{what}] max_abs_err={err.max().item():.3e} max_ref={ref.abs().max().item():.3e} frac_out_of_tol={frac:.2e}")
    assert frac == 0.0, f"{what}: {frac:.3e} of elements out of tolerance, max err {err.max().item():.3e}"


# ------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,tile_n", [
    (128, 128, 64, 128),
    (256, 256, 128, 64),
    (256, 256, 256, 256),
    (2048, 1280, 1280, 0),
    (154, 640, 2048, 0),      # text K/V projection rows (B*77), M not a multiple of 128
    (8192, 320, 320, 128),    # N = 2.5 tiles
    (1000, 1920, 640, 0),
    (300, 72, 200, 64),       # K not a multiple of 64 (TMA zero-fill), N not a multiple of 64
    (256, 256, 64, 512),      # widest tile request (256 columns), single k-block
    (2048, 1280, 1280, 512),  # persistent over several tiles
    (8192, 640, 2560, 512),   # partially filled N tile (640 = 2.5 x 256)
    (384, 3840, 1280, 512),   # odd number of 128-row tiles
    (1000, 1920, 640, 512),
    (2048, 1280, 1280, 192),  # 128x192 tiles: 7 N tiles, the last one clipped at N
    (300, 200, 320, 192),
    (2048, 1280, 5120, 384),  # 192-column tile request, long K
    (384, 1280, 640, 384),    # 192-column tile, odd number of 128-row tiles, clipped last N tile
    (1000, 200, 320, 384),
    (2048, 1280, 5120, 0),    # library's choice for long K
    (512, 1280, 1280, 64),    # 128x64 tiles: the 1280-channel level of a 512^2 edit (80 tiles instead of 28)
    (512, 1280, 5120, 64),
])
def test_gemm_plain(ops, M, N, K, tile_n):
    x = rnd(M, K)
    w = rnd(N, K, scale=K ** -0.5)
    out = ops.linear(x, w, tile_n=tile_n)
    torch.cuda.synchronize()
    check(out, x.float() @ w.float().t(), f"gemm {M}x{N}x{K} bn{tile_n}")


def test_gemm_epilogues(ops):
    M, N, K = 2048, 640, 1280
    x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N)
    res = rnd(M, N, seed=3)
    rb = rnd(2, N, seed=5)
    base = x.float() @ w.float().t()
    check(ops.linear(x, w, b), base + b.float(), "gemm+bias")
    check(ops.linear(x, w, b, residual=res), base + b.float() + res.float(), "gemm+bias+res")
    ref = base + b.float() + rb.float().repeat_interleave(M // 2, dim=0)
    check(ops.linear(x, w, b, rowbias=rb, rows_per_group=M // 2), ref, "gemm+bias+rowbias")
    check(ops.linear(x, w, b, silu=True), F.silu(base + b.float()), "gemm+bias+silu")
    # strided input / output views (fused QKV style buffers)
    big = rnd(M, 3 * K, seed=7)
    xv = big[:, K:2 * K]
    obuf = torch.zeros(M, 2 * N, dtype=torch.float16, device="cuda")
    ops.linear(xv, w, out=obuf[:, N:])
    check(obuf[:, N:], xv.float() @ w.float().t(), "gemm strided in/out")
    assert (obuf[:, :N] == 0).all()


@pytest.mark.parametrize("tile_n", [256, 512])
@pytest.mark.parametrize("M,C", [(2048, 1280), (512, 640), (100, 640)])
def test_gemm_geglu(ops, M, C, tile_n):
    x = rnd(M, C)
    w = rnd(8 * C, C, scale=C ** -0.5)
    b = rnd(8 * C)
    out = ops.linear(x, w, b, geglu=True, tile_n=tile_n)
    h = x.float() @ w.float().t() + b.float()
    a, g = h.chunk(2, dim=-1)
    check(out, a * F.gelu(g), f"geglu {M}x{C}")


@pytest.mark.parametrize("M,N,K,geglu,tile_n", [
    (2048, 3840, 1280, False, 0),     # norm1 -> q|k|v
    (2048, 1280, 1280, False, 192),
    (8192, 640, 640, False, 0),       # norm2 -> to_q at the 640-channel level
    (2048, 5120, 1280, True, 0),      # norm3 -> GEGLU projection
    (1000, 2560, 640, True, 512),     # widest tile request, ragged M
    (512, 1280, 1280, False, 64),     # 128x64 tiles, producer (bias + residual + statistics) and consumer
    (2048, 3840, 1280, False, 512),   # q|k|v consumer on the widest tile
])
def test_gemm_layernorm_fold(ops, M, N, K, geglu, tile_n):
    """producer GEMM writes per-row (sum, sumsq) slabs; the consumer applies LayerNorm algebraically in its epilogue."""
    a = rnd(M, K, seed=31)
    wp = rnd(K, K, scale=K ** -0.5, seed=32)
    bp = rnd(K, seed=33)
    res = rnd(M, K, seed=34) * 2 + 0.5            # non-zero mean rows
    stats = torch.full(((K + 63) // 64, M, 2), float("nan"), dtype=torch.float32, device="cuda")
    h = ops.linear(a, wp, bp, residual=res, stats_out=stats, tile_n=64 if tile_n == 64 else 0)
    hf = h.float()
    # the statistics are those of the ROUNDED fp16 output rows
    s = stats.sum(dim=0)
    torch.testing.assert_close(s[:, 0], hf.sum(dim=1), rtol=1e-5, atol=1e-3)
    torch.testing.assert_close(s[:, 1], (hf * hf).sum(dim=1), rtol=1e-5, atol=1e-3)

    gamma = (1 + 0.2 * rnd(K, seed=35).float()).half()
    beta = (0.1 * rnd(K, seed=36).float()).half()
    rows = 2 * N if geglu else N
    w = rnd(rows, K, scale=K ** -0.5, seed=37)
    b = rnd(rows, scale=0.25, seed=38)
    w_c, c = ops.fold_layernorm(w, b, gamma, beta)
    out = ops.linear(h, w_c, c, geglu=geglu, ln=(stats, 1e-5), tile_n=tile_n)
    # exact (fp64) result, and the unfused kernel pipeline (explicit LayerNorm kernel -> GEMM) the fold replaces
    n64 = F.layer_norm(h.double(), (K,), gamma.double(), beta.double(), 1e-5)
    y = n64 @ w.double().t() + b.double()
    exact = (y[:, :N] * F.gelu(y[:, N:]) if geglu else y).float()
    unfused = ops.linear(ops.layernorm(h, gamma, beta, 1e-5), w, b, geglu=geglu).float()
    e_fold, e_unf = (out.float() - exact).abs(), (unfused - exact).abs()
    rms_fold, rms_unf = e_fold.pow(2).mean().sqrt().item(), e_unf.pow(2).mean().sqrt().item()
    print(f"[ln_fold M{M} N{N} K{K} geglu{geglu}] rms err fold {rms_fold:.3e} unfused {rms_unf:.3e}; "
          f"max fold {e_fold.max().item():.3e} unfused {e_unf.max().item():.3e}")
    # the fold moves one fp16 rounding from LN(x) to W*gamma and rounds c = W beta + b to fp16 once more (<= ulp(c)/2):
    # it must stay in the accuracy class of the pipeline it replaces
    assert torch.isfinite(out).all()
    assert rms_fold <= 1.5 * rms_unf + 1e-6, (rms_fold, rms_unf)
    assert e_fold.max().item() <= 2.0 * e_unf.max().item() + 1e-3
    if not geglu:
        check(out, exact, f"ln_fold M{M} N{N} K{K}", rtol=2e-3, atol=2e-3)


# ------------------------------------------------------------------------------------------------------------
# conv 3x3
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [
    (2, 32, 32, 64, 128, 1),
    (1, 16, 16, 128, 64, 1),
    (2, 32, 32, 1280, 1280, 1),
    (2, 128, 128, 320, 320, 1),
    (2, 64, 64, 960, 640, 1),
    (2, 24, 24, 128, 128, 1),    # 768^2 level-2 spatial size (tile does not divide)
    (2, 96, 96, 64, 64, 1),
    (2, 32, 32, 128, 128, 2),
    (2, 128, 128, 320, 320, 2),
])
def test_conv3x3(ops, B, H, W, Cin, Cout, stride):
    x_nchw = rnd(B, Cin, H, W)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rnd(Cout)
    x = x_nchw.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, stride=stride)
    ref = F.conv2d(x_nchw.float(), w.float(), b.float(), stride=stride, padding=1).permute(0, 2, 3, 1)
    check(out, ref, f"conv3x3 {B}x{H}x{W} {Cin}->{Cout} s{stride}")


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [
    (2, 32, 32, 1280, 1280, 1), (2, 64, 64, 640, 640, 1), (1, 24, 24, 128, 320, 1), (2, 64, 64, 320, 320, 2),
])
@pytest.mark.parametrize("tile_n", [512, 192, 384, 64])
def test_conv3x3_tile_variants(ops, B, H, W, Cin, Cout, stride, tile_n):
    x_nchw = rnd(B, Cin, H, W)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rnd(Cout)
    res = rnd(B, H // stride, W // stride, Cout, seed=21)
    x = x_nchw.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, stride=stride, residual=res, tile_n=tile_n)
    ref = F.conv2d(x_nchw.float(), w.float(), b.float(), stride=stride, padding=1).permute(0, 2, 3, 1) + res.float()
    check(out, ref, f"conv3x3 bn{tile_n} {B}x{H}x{W} {Cin}->{Cout} s{stride}")


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [
    (2, 32, 32, 1280, 1280, 1),
])
def test_conv3x3_cta_pair(ops, B, H, W, Cin, Cout, stride):
    x_nchw = rnd(B, Cin, H, W)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rnd(Cout)
    x = x_nchw.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, stride=stride, tile_n=512)
    ref = F.conv2d(x_nchw.float(), w.float(), b.float(), stride=stride, padding=1).permute(0, 2, 3, 1)
    check(out, ref, f"conv3x3 pair {B}x{H}x{W} {Cin}->{Cout} s{stride}")


def test_conv3x3_epilogue(ops):
    B, H, W, Cin, Cout = 2, 32, 32, 128, 256
    x_nchw = rnd(B, Cin, H, W)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rnd(Cout)
    temb = rnd(B, 512, seed=11)          # a slice of a wider time-embedding buffer
    res = rnd(B, H, W, Cout, seed=13)
    x = x_nchw.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), b, rowbias=temb[:, 128:128 + Cout], residual=res)
    ref = F.conv2d(x_nchw.float(), w.float(), b.float(), padding=1).permute(0, 2, 3, 1)
    ref = ref + temb[:, 128:128 + Cout].float()[:, None, None, :] + res.float()
    check(out, ref, "conv3x3+temb+res")


# ------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------
def sdpa_ref(q, k, v, B, H, Nq, Nk):
    qf = q.float().view(B, Nq, H, 64).transpose(1, 2)
    kf = k.float().view(B, Nk, H, 64).transpose(1, 2)
    vf = v.float().view(B, Nk, H, 64).transpose(1, 2)
    s = qf @ kf.transpose(-1, -2) / 8.0
    o = s.softmax(-1) @ vf
    return o.transpose(1, 2).reshape(B * Nq, H * 64)


@pytest.mark.parametrize("B,H,Nq,Nk", [
    (1, 1, 128, 128),
    (2, 4, 256, 256),
    (2, 20, 1024, 1024),
    (2, 10, 4096, 4096),
    (2, 5, 576, 576),      # 768^2: tail q tile and tail kv block
    (2, 4, 1024, 77),      # text-only cross attention (skip=True layers)
    (1, 2, 100, 300),
])
def test_attention(ops, B, H, Nq, Nk):
    q, k, v = rnd(B * Nq, H * 64), rnd(B * Nk, H * 64, seed=1), rnd(B * Nk, H * 64, seed=2)
    out = ops.attention(q, k, v, B, H, Nq, Nk)
    check(out, sdpa_ref(q, k, v, B, H, Nq, Nk), f"attn B{B} H{H} {Nq}x{Nk}")


@pytest.mark.parametrize("B,H,Nq,Nk,qscale", [
    (2, 20, 1024, 1024, 1.0),   # 320 query tiles: the partial last wave is cut into KV parts
    (2, 10, 4096, 4096, 1.0),   # 640 query tiles, 32 KV blocks each
    (2, 5, 576, 576, 3.0),      # ragged: partial last query tile, clipped last KV block, very different part maxima
    (1, 3, 2000, 1500, 2.0),
])
def test_attention_kv_split(ops, B, H, Nq, Nk, qscale):
    """the KV-split plan (partial O, m, l -> merge kernel) must agree with whole-tile processing and the reference."""
    q, k, v = rnd(B * Nq, H * 64, scale=qscale), rnd(B * Nk, H * 64, seed=1), rnd(B * Nk, H * 64, seed=2)
    from imagharmony_b200 import _lib
    lib = _lib.load()
    lib.ih_attention_set_split_policy(1)       # split even where the cost model would not bother
    try:
        assert lib.ih_attention_workspace_bytes(B, H, Nq, Nk, 0) > 0, "shape does not exercise the split path"
        whole = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=False)
        split = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=True)
        again = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=True)
    finally:
        lib.ih_attention_set_split_policy(0)
    ref = sdpa_ref(q, k, v, B, H, Nq, Nk)
    check(whole, ref, f"attn whole B{B} H{H} {Nq}x{Nk}")
    check(split, ref, f"attn kv-split B{B} H{H} {Nq}x{Nk}")
    assert torch.equal(split, again), "KV-split attention must be run-to-run deterministic"


def test_attention_fused_qkv_views(ops):
    B, H, N = 2, 10, 512
    C = H * 64
    qkv = rnd(B * N, 3 * C)
    out = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, H, N, N)
    check(out, sdpa_ref(qkv[:, :C].contiguous(), qkv[:, C:2 * C].contiguous(), qkv[:, 2 * C:].contiguous(), B, H, N, N),
          "attn fused qkv views")


@pytest.mark.parametrize("scale", [1.0, 0.7, 0.0])
@pytest.mark.parametrize("Nq", [1024, 256, 576])
def test_attention_decoupled_ip(ops, Nq, scale):
    """out = SDPA(q, k_t, v_t) + scale * SDPA(q, k_ip, v_ip): attention_processor.py:423-450."""
    B, H, Nt, Ni = 2, 20, 77, 4
    C = H * 64
    q = rnd(B * Nq, C)
    k = rnd(B * (Nt + Ni), C, seed=1)
    v = rnd(B * (Nt + Ni), C, seed=2)
    out = ops.attention(q, k, v, B, H, Nq, Nt + Ni, n_ip=Ni, ip_scale=scale)
    k3, v3 = k.view(B, Nt + Ni, C), v.view(B, Nt + Ni, C)
    ref_t = sdpa_ref(q, k3[:, :Nt].reshape(-1, C), v3[:, :Nt].reshape(-1, C), B, H, Nq, Nt)
    ref_i = sdpa_ref(q, k3[:, Nt:].reshape(-1, C), v3[:, Nt:].reshape(-1, C), B, H, Nq, Ni)
    check(out, ref_t + scale * ref_i, f"decoupled ip attn Nq{Nq} s{scale}")


def test_attention_decoupled_ip_long_text(ops):
    """96 < Nk <= 128 with image tokens: one 128-key block, two-segment softmax (attn_f16_kernel)."""
    B, H, Nq, Nt, Ni = 2, 4, 300, 100, 16
    C = H * 64
    q, k, v = rnd(B * Nq, C), rnd(B * (Nt + Ni), C, seed=1), rnd(B * (Nt + Ni), C, seed=2)
    out = ops.attention(q, k, v, B, H, Nq, Nt + Ni, n_ip=Ni, ip_scale=0.5)
    k3, v3 = k.view(B, Nt + Ni, C), v.view(B, Nt + Ni, C)
    ref_t = sdpa_ref(q, k3[:, :Nt].reshape(-1, C), v3[:, :Nt].reshape(-1, C), B, H, Nq, Nt)
    ref_i = sdpa_ref(q, k3[:, Nt:].reshape(-1, C), v3[:, Nt:].reshape(-1, C), B, H, Nq, Ni)
    check(out, ref_t + 0.5 * ref_i, "decoupled ip attn Nk=116")


# ------------------------------------------------------------------------------------------------------------
# norms
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,C,silu", [(2, 32, 1280, True), (2, 128, 320, True), (2, 64, 640, False), (1, 24, 960, True)])
def test_groupnorm(ops, B, H, C, silu):
    x = (rnd(B, H, H, C) * 2 + 0.5).half()
    g, b = rnd(C) + 1, rnd(C, seed=1)
    eps = 1e-5 if silu else 1e-6
    out = ops.groupnorm(x, g, b, eps=eps, silu=silu)
    ref = F.group_norm(x.float().permute(0, 3, 1, 2), 32, g.float(), b.float(), eps)
    if silu:
        ref = F.silu(ref)
    check(out, ref.permute(0, 2, 3, 1), f"groupnorm {B}x{H}x{C}", rtol=2e-3, atol=2e-3)


def test_groupnorm_concat(ops):
    B, H, C0, C1 = 2, 32, 1280, 640
    x0, x1 = rnd(B, H, H, C0), rnd(B, H, H, C1, seed=4) * 3
    g, b = rnd(C0 + C1) + 1, rnd(C0 + C1, seed=1)
    out = ops.groupnorm(x0, g, b, x1=x1, silu=True)
    xc = torch.cat([x0, x1], -1).float().permute(0, 3, 1, 2)
    ref = F.silu(F.group_norm(xc, 32, g.float(), b.float(), 1e-5)).permute(0, 2, 3, 1)
    check(out, ref, "groupnorm concat", rtol=2e-3, atol=2e-3)
    cat = ops.concat_channels(x0, x1)
    assert torch.equal(cat, torch.cat([x0, x1], -1))


@pytest.mark.parametrize("rows,C", [(2048, 1280), (8192, 640), (8, 2048), (3, 4096)])
def test_layernorm(ops, rows, C):
    x = (rnd(rows, C) * 3 + 1).half()
    g, b = rnd(C) + 1, rnd(C, seed=1)
    out = ops.layernorm(x, g, b, 1e-5)
    check(out, F.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5), f"layernorm {rows}x{C}", rtol=2e-3, atol=2e-3)


# ------------------------------------------------------------------------------------------------------------
# small kernels
# ------------------------------------------------------------------------------------------------------------
def test_linear_small(ops):
    x = rnd(2, 2816)
    w, b = rnd(1280, 2816, scale=2816 ** -0.5), rnd(1280)
    check(ops.linear_small(x, w, b), x.float() @ w.float().t() + b.float(), "linear_small")
    check(ops.linear_small(x, w, b, act_out=True), F.silu(x.float() @ w.float().t() + b.float()), "linear_small silu out",
          rtol=2e-3, atol=2e-3)
    check(ops.linear_small(x, w, b, act_in=True), F.silu(x.float()).half().float() @ w.float().t() + b.float(),
          "linear_small silu in")


def test_sinusoid(ops):
    t = torch.tensor([981.0, 1.0, 500.0], device="cuda")
    out = ops.sinusoid(t, 320, 3)
    half = 160
    f = torch.exp(-math.log(10000.0) * torch.arange(half, device="cuda").float() / half)
    a = t[:, None] * f[None]
    check(out, torch.cat([a.cos(), a.sin()], -1), "sinusoid", rtol=2e-3, atol=2e-3)
    step = torch.tensor([2], dtype=torch.int32, device="cuda")
    out2 = ops.sinusoid(t, 320, 2, step=step)
    assert torch.equal(out2[0], out[2]) and torch.equal(out2[1], out[2])


def test_upsample(ops):
    x = rnd(2, 16, 16, 64)
    out = ops.upsample2x(x)
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(out.float(), ref)


def test_euler_cfg_step(ops):
    n, H = 2, 64
    lat = rnd(n, 4, H, H) * 5
    noise = rnd(2 * n, 4, H, H, seed=2)
    sig = torch.tensor([13.1204, 11.6761, 10.4250, 0.0], device="cuda")
    step = torch.tensor([1], dtype=torch.int32, device="cuda")
    model_in = torch.empty(2 * n, 4, H, H, dtype=torch.float16, device="cuda")
    lat_ref = lat.clone()
    ops.euler_cfg_step(noise, lat, model_in, sig, step, 5.0)
    u, c = noise.chunk(2)
    eps = u + 5.0 * (c - u)            # fp16 tensor arithmetic like custom_pipelines.py:348-350
    x = lat_ref.float()
    x0 = x - (sig[1] * eps.float()).half().float()   # diffusers: 0-dim fp32 sigma * fp16 tensor -> fp16 product
    d = (x - x0) / sig[1]
    xn = (x + d * (sig[2] - sig[1])).half()
    assert int(step.item()) == 2
    check(lat, xn, "euler latents", rtol=1e-3, atol=1e-3)
    mi = (xn.float() / (sig[2] ** 2 + 1) ** 0.5).half()
    check(model_in, torch.cat([mi, mi]), "euler model_in")
    m2 = torch.empty_like(model_in)
    ops.scale_model_input(lat, m2, sig, step)
    check(m2, torch.cat([mi, mi]), "scale_model_input")


# latent sizes of SDXL buckets (832x1216, 640x1536, 768x1344): the per-image rescale reduction over 4*h*w elements that
# are not a power of two
STEP_BUCKETS = [(104, 152), (80, 192), (96, 168)]


@pytest.mark.parametrize("use_cfg,rescale,n,h,w", [
    pytest.param(False, 0.0, 3, 64, 64, id="False-0.0"),
    pytest.param(True, 0.7, 3, 64, 64, id="True-0.7"),
    pytest.param(True, 1.0, 3, 64, 64, id="True-1.0"),
] + [pytest.param(True, 0.7, n, h, w, id=f"True-0.7-n{n}-{h}x{w}") for n in (1, 3) for h, w in STEP_BUCKETS])
def test_euler_step_ex(ops, use_cfg, rescale, n, h, w):
    """ih_euler_step_ex: no-CFG (custom_pipelines.py:223) and guidance_rescale (:352-354) variants of the transition,
    against the fp16 tensor arithmetic of the reference loop (oracle/scheduler_ref.py rescale_noise_cfg)."""
    from oracle.scheduler_ref import rescale_noise_cfg
    b = 2 * n if use_cfg else n
    lat = rnd(n, 4, h, w) * 5
    noise = rnd(b, 4, h, w, seed=2)
    sig = torch.tensor([13.1204, 11.6761, 10.4250, 0.0], device="cuda")
    step = torch.tensor([1], dtype=torch.int32, device="cuda")
    model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
    lat_ref = lat.clone()
    ops.euler_step(noise, lat, model_in, sig, step, 5.0, use_cfg=use_cfg, guidance_rescale=rescale)
    if use_cfg:
        u, c = noise.chunk(2)
        eps = u + 5.0 * (c - u)
        eps = rescale_noise_cfg(eps, c, rescale)          # fp16 tensors -> fp16 rounding points
    else:
        eps = noise
    x = lat_ref.float()
    x0 = x - (sig[1] * eps.float()).half().float()
    xn = (x + (x - x0) / sig[1] * (sig[2] - sig[1])).half()
    assert int(step.item()) == 2
    # sigma ~ 11.7 amplifies one fp16 ulp of eps (the std ratio is itself an fp16 number): 2e-3 relative on |x| ~ 20
    check(lat, xn, f"euler_ex latents cfg={use_cfg} r={rescale}", rtol=2e-3, atol=2e-3)
    mi = (lat.float() / (sig[2] ** 2 + 1) ** 0.5).half()
    check(model_in, torch.cat([mi, mi]) if use_cfg else mi, "euler_ex model_in")
    m2 = torch.empty_like(model_in)
    ops.scale_model_input(lat, m2, sig, step, duplicate=use_cfg)
    check(m2, torch.cat([mi, mi]) if use_cfg else mi, "scale_model_input_ex")


@pytest.mark.parametrize("B,H,W,Cin,Cout,C0,C1", [(2, 32, 32, 128, 192, 64, 0), (2, 16, 16, 256, 128, 192, 64),
                                                   (1, 24, 40, 64, 320, 128, 192), (2, 32, 32, 1280, 1280, 1280, 1280)])
def test_conv3x3_fused_shortcut(ops, B, H, W, Cin, Cout, C0, C1):
    """conv2(h) + conv_shortcut(cat(x, skip)) of a ResnetBlock2D as ONE implicit-GEMM launch (extra K blocks over one or two
    further NHWC sources) against conv2d + 1x1 conv in fp32."""
    h = rnd(B, H, W, Cin, seed=1)
    w3 = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    x0 = rnd(B, H, W, C0, seed=3)
    x1 = rnd(B, H, W, C1, seed=4) if C1 else None
    wsc = rnd(Cout, C0 + C1, scale=(C0 + C1) ** -0.5, seed=5)
    bias = rnd(Cout, seed=6)
    temb = rnd(B, Cout, seed=7)
    w_ext = torch.cat([ops.pack_conv3x3_weight(w3), wsc], dim=1).contiguous()
    out = ops.conv3x3(h, w_ext, bias, rowbias=temb, shortcut=(x0, x1))
    src = x0 if x1 is None else torch.cat([x0, x1], dim=-1)
    ref = (F.conv2d(h.float().permute(0, 3, 1, 2), w3.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
           + src.float() @ wsc.float().t() + temb.float()[:, None, None, :])
    check(out, ref, f"conv3x3 + fused shortcut {Cin}->{Cout} sc {C0}+{C1}")
