"""The tensor-core GEMM and the implicit-GEMM 3x3 convolution in exact arithmetic (tests/exact_gemm.py): small-integer
operands, so every output is held bit for bit to fp16 of the fp64 reference -- or, behind the LayerNorm fold's rsqrtf
and the transcendental activations, to 1 fp16 ulp of it -- on every tile width, ring position, K tail, epilogue
combination, spatial tile and entry point, with NaN and sentinels around every operand and output window."""
import pytest
import torch

import exact_gemm as E

pytestmark = pytest.mark.gpu

WORST = {}   # epilogue -> largest err / bar seen (printed at the end of the module)


@pytest.fixture(scope="module")
def ops():
    torch.backends.cuda.matmul.allow_tf32 = False
    from imagharmony_b200 import ops as _ops
    yield _ops
    print("\n[exact_gemm] largest err / 1-ulp bar per non-exact epilogue:",
          {k: round(v, 3) for k, v in sorted(WORST.items())})


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def window(t, left, right, fill):
    """t as the column window [:, left:left + cols] of a wider buffer holding `fill` elsewhere, and a trailing row."""
    M, n = t.shape
    buf = torch.full((M + 1, left + n + right), fill, dtype=t.dtype, device=t.device)
    buf[:M, left:left + n] = t
    return buf, buf[:M, left:left + n]


def run_gemm(ops, c, tile_n):
    """One launch of case c: A a window of a NaN-filled buffer, the residual a window with NaN on both sides, the
    output a window with sentinels on both sides and below, which must stay untouched.  Returns the output."""
    M, K = c["M"], c["K"]
    n_out = c["N"] // 2 if c["geglu"] else c["N"]
    _, a = window(c["a"], 64, 24, float("nan"))
    res = None
    if "residual" in c:
        _, res = window(c["residual"], 8, 8, float("nan"))
    obuf, out = window(torch.zeros(M, n_out, dtype=torch.float16, device="cuda"), 8, 16, E.SENTINEL)
    stats = None
    if c["stats"]:
        stats = torch.full((-(-n_out // 64), M, 2), float("nan"), dtype=torch.float32, device="cuda")
        c["stats_out"] = stats
    ops.linear(a, c["w"], c.get("bias"), residual=res, rowbias=c.get("rowbias"), rows_per_group=c["rows_per_group"],
               geglu=c["geglu"], silu=c["act"] == "silu", gelu=c["act"] == "gelu",
               quick_gelu=c["act"] == "quick_gelu", out=out, tile_n=tile_n,
               ln=(c["ln_stats"], c["eps"]) if c["ln"] else None, stats_out=stats, alpha=c["alpha"], relu=c["relu"])
    torch.cuda.synchronize()
    around = obuf.clone()
    around[:M, 8:8 + n_out] = E.SENTINEL
    assert bool((around == E.SENTINEL).all()), "a store left the output window"
    return out


def check_gemm(ops, c, tile_n, what, bn_out=None):
    ref, pre = E.gemm_ref(c)
    E.gemm_check_bounds(c, ref, pre)
    out = run_gemm(ops, c, tile_n)
    bad, r = E.gemm_bar(out, c, ref)
    if bad is not None:
        assert bad == 0, (what, E.first_mismatch(out, ref, bn_out))
    else:
        key = ("ln+" if c["ln"] else "") + ("geglu" if c["geglu"] else (c["act"] or "ln"))
        WORST[key] = max(WORST.get(key, 0.0), r)
        assert r <= 1.0, (what, r)
    if c["stats"]:
        st = c["stats_out"]
        assert E.stats_bad(st, out) == 0, (what, "stats_out slot totals differ from the exact row sums")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# gemm_f16_kernel: every tile at every ring position
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geglu,bn,stages,kb,per_cta,tail", E.ring_cases(),
                         ids=[f"{'geglu' if g else 'plain'}{bn}-kb{kb}-cta{p}-tail{t}"
                              for g, bn, _, kb, p, t in E.ring_cases()])
def test_ring_positions(ops, geglu, bn, stages, kb, per_cta, tail):
    M, N, K = E.ring_shape(geglu, bn, kb, per_cta, tail, sms())
    c = E.gemm_case(M, N, K, seed=bn + kb, bias=True, geglu=geglu, device="cuda")
    check_gemm(ops, c, bn, (geglu, bn, kb, per_cta), bn // 2 if geglu else bn)


# ---------------------------------------------------------------------------------------------------------------------
# every epilogue combination on every tile
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", sorted(E.PLAIN_STAGES))
@pytest.mark.parametrize("i,name", list(enumerate(n for n, _ in E.PLAIN_EPILOGUES)))
def test_plain_epilogues(ops, bn, i, name):
    kw = dict(E.PLAIN_EPILOGUES[i][1])
    M, N, K, rpg = E.epilogue_shape(False, bn, i)
    c = E.gemm_case(M, N, K, seed=7 * i + bn, rows_per_group=rpg, device="cuda", **kw)
    check_gemm(ops, c, bn, (bn, name), bn)


@pytest.mark.parametrize("bn", sorted(E.GEGLU_STAGES))
@pytest.mark.parametrize("i,name", list(enumerate(n for n, _ in E.GEGLU_EPILOGUES)))
def test_geglu_epilogues(ops, bn, i, name):
    kw = dict(E.GEGLU_EPILOGUES[i][1])
    if bn == 192 and kw.get("stats"):
        pytest.skip("the 192-row GEGLU tile refuses stats_out (a 96-output tile would split a 64-column slot)")
    M, N, K, rpg = E.epilogue_shape(True, bn, i)
    c = E.gemm_case(M, N, K, seed=11 * i + bn, geglu=True, bias=True, rows_per_group=rpg, device="cuda", **kw)
    check_gemm(ops, c, bn, (bn, name), bn // 2)


@pytest.mark.parametrize("bn", E.SCALED_TILES)
@pytest.mark.parametrize("i,name", list(enumerate(n for n, _ in E.SCALED_EPILOGUES)))
def test_scaled_epilogues(ops, bn, i, name):
    """alpha = 2^-k, ReLU after the residual: ih_gemm_scaled_f16 takes no tile width, so the shape makes the cost
    model choose each tile (exact_gemm.scaled_shape restates pick_bn)."""
    if sms() != E.NUM_SMS:
        pytest.skip("the shapes are chosen for 132 SMs")
    M, N, K = E.scaled_shape(bn)
    c = E.gemm_case(M, N, K, seed=13 * i + bn, device="cuda", **E.SCALED_EPILOGUES[i][1])
    check_gemm(ops, c, 0, (bn, name), bn)


@pytest.mark.parametrize("name,M,N,K,kw", E.SDXL_AUTO, ids=[s[0] for s in E.SDXL_AUTO])
def test_sdxl_shapes_library_choice(ops, name, M, N, K, kw):
    """tile_n = 0 at SDXL UNet / refiner / VAE launch shapes: whichever kernel and tile the library picks."""
    kw = dict(kw)
    if kw.get("geglu"):
        kw["bias"] = True
    c = E.gemm_case(M, N, K, seed=len(name), rows_per_group=4096 if kw.get("rowbias") else 0, device="cuda", **kw)
    check_gemm(ops, c, 0, name)


@pytest.mark.parametrize("qkv_tile", [0, 1])
def test_stats_chain_feeds_layernorm_fold(ops, qkv_tile):
    """attn-out -> q|k|v and -> GEGLU: the statistics one GEMM writes (160-column tiles: the carry into slots 3 and 4)
    are the ln= input of the next, as in a transformer block.  The consumers are held to 1 ulp of the fp64 LayerNorm
    fold of the producer's exact output."""
    M, C = 2 * 1024 - 40, 640
    prod = E.gemm_case(M, C, C, seed=21, bias=True, residual=True, stats=True, device="cuda")
    prod["w"] = E.sparse_rows(C, C, 4, 22, "cuda")            # |x| small: row std ~ 1, rstd in the 4-bar range
    x = check_gemm(ops, prod, 160, "producer", 160)
    st = prod["stats_out"]
    for geglu, N in ((False, 3 * C), (True, 8 * C)):
        cons = E.gemm_case(M, N, C, seed=23 + geglu, ln=True, bias=geglu, geglu=geglu, device="cuda")
        cons["a"] = x.clone()
        cons["ln_stats"] = E.slab_stats(x)
        assert torch.equal(cons["ln_stats"].sum(0), st.sum(0)), "slot totals of the producer"
        cons["ln_stats"] = st       # the real producer's slots, as the block passes them
        want, pre = E.gemm_ref(cons)
        E.gemm_check_bounds(cons, want, pre)
        got = torch.empty(M, N // 2 if geglu else N, dtype=torch.float16, device="cuda")
        ops.linear(x, cons["w"], cons.get("bias"), geglu=geglu, ln=(st, cons["eps"]),
                   tile_n=ops.TILE_PINGPONG if qkv_tile else 0, out=got)
        r = E.ratio(got, want, 1.0, cons["slack"])
        WORST["ln+chain"] = max(WORST.get("ln+chain", 0.0), r)
        assert r <= 1.0, (geglu, r)


def test_premise_cublas_integer_matmul_is_exact():
    """The hardware premise: cuBLAS's fp16 GEMM (no reduced-precision reduction) of the same integer operands gives
    fp16 of the fp64 product.  If a kernel case fails and this passes, the kernel is wrong."""
    old = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    try:
        for M, N, K in ((1000, 1480, 1288), (2048, 1280, 5120), (777, 328, 8)):
            a, w = E.dense(M, K, 1, 1, "cuda"), E.dense(N, K, 2, 1, "cuda")
            want = a.double() @ w.double().t()
            assert float(want.abs().max()) <= 2048
            assert torch.equal(torch.matmul(a, w.t()), want.half())
    finally:
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = old


# ---------------------------------------------------------------------------------------------------------------------
# 3x3 convolution: every entry point at SDXL's latent levels, every spatial tile, every forced tile width
# ---------------------------------------------------------------------------------------------------------------------
def poisoned_images(t, fill):
    """t [B, ...] as the first B images of a buffer whose image B is `fill`."""
    buf = torch.full((t.shape[0] + 1,) + tuple(t.shape[1:]), fill, dtype=t.dtype, device=t.device)
    buf[:t.shape[0]] = t
    return buf[:t.shape[0]]


def run_conv(ops, entry, x, w, *, bias=None, rowbias=None, residual=None, alpha=1.0, relu=False, shortcut=(),
             stride=1, tile_n=0):
    B, H, W, _ = x.shape
    Ho, Wo = H // stride, W // stride
    obuf = torch.full((B + 1, Ho, Wo, w.shape[0]), E.SENTINEL, dtype=torch.float16, device="cuda")
    out = obuf[:B]
    x = poisoned_images(x, float("nan"))
    if residual is not None:
        residual = poisoned_images(residual, float("nan"))
    sc = [poisoned_images(s, float("nan")) for s in shortcut]
    if entry == "down":
        ops.conv3x3_down(x, w, bias, out=out, tile_n=tile_n, alpha=alpha)
    elif entry == "shortcut":
        ops.conv3x3(x, w, bias, rowbias=rowbias, shortcut=(sc[0], sc[1] if len(sc) > 1 else None), out=out)
    else:
        ops.conv3x3(x, w, bias, rowbias=rowbias, residual=residual, stride=stride, out=out, tile_n=tile_n,
                    alpha=alpha, relu=relu)
    torch.cuda.synchronize()
    assert bool((obuf[B] == E.SENTINEL).all()), "a store left the output"
    return out


# (entry, stride, kwargs): ih_conv2d_f16 with bias + row bias + residual and at stride 2; ih_conv2d_scaled_f16 with
# and without ReLU; ih_conv2d_shortcut_f16 with one and two sources; ih_conv2d_down_f16
CONV_ENTRIES = [
    ("conv", 1, dict(bias=True, rowbias=True, residual=True)),
    ("conv", 2, dict(bias=True)),
    ("scaled", 1, dict(alpha=0.5, bias=True, residual=True)),
    ("scaled_relu", 2, dict(alpha=0.25, relu=True, bias=True, residual=True)),
    ("shortcut", 1, dict(bias=True, rowbias=True, sources=1)),
    ("shortcut", 1, dict(bias=True, sources=2)),
    ("down", 2, dict(alpha=0.5, bias=True)),
]


def conv_case(ops, entry, stride, kw, B, H, W, Cin, Cout, seed, selector=False, tile_n=0):
    if stride == 2 and (H % 2 or W % 2):
        H, W = 2 * H, 2 * W
    Ho, Wo = H // stride, W // stride
    x = E.conv_input(B, H, W, Cin, seed, "cuda")
    shortcut = []
    if kw.get("sources"):
        chans = [Cin, 64 * max(1, Cin // 128)][:kw["sources"]]
        shortcut = [E.conv_input(B, H, W, ch, seed + 1 + i, "cuda") for i, ch in enumerate(chans)]
    K = 9 * Cin + sum(s.shape[-1] for s in shortcut)
    if selector:
        w, _ = E.selector_weight(Cout, Cin, [s.shape[-1] for s in shortcut], seed, "cuda")
    else:
        w = E.conv_weight(Cout, K, seed + 3, "cuda")
    bias = E.vec(Cout, -3, 3, seed + 4, "cuda") if kw.get("bias") else None
    rowbias = E.ints(B + 1, Cout, -3, 3, seed + 5, "cuda").half() if kw.get("rowbias") else None
    residual = E.ints(B * Ho * Wo, Cout, -4, 4, seed + 6, "cuda").half().view(B, Ho, Wo, Cout) \
        if kw.get("residual") else None
    alpha, relu = kw.get("alpha", 1.0), kw.get("relu", False)
    ref = E.conv_ref(x, w, stride=stride, pad="br" if entry == "down" else "all", bias=bias,
                     rowbias=None if rowbias is None else rowbias[:B], residual=residual, alpha=alpha, relu=relu,
                     shortcut=shortcut)
    E.conv_check_bounds(x, w, ref, shortcut)
    out = run_conv(ops, "down" if entry == "down" else ("shortcut" if shortcut else "conv"), x, w, bias=bias,
                   rowbias=None if rowbias is None else rowbias[:B], residual=residual, alpha=alpha, relu=relu,
                   shortcut=shortcut, stride=stride, tile_n=tile_n)
    assert E.check_bits(out, ref) == 0, (entry, stride, B, H, W, Cin, Cout, selector, tile_n,
                                         E.first_mismatch(out.reshape(-1, Cout), ref.reshape(-1, Cout)))


@pytest.mark.parametrize("selector", [False, True])
@pytest.mark.parametrize("j", range(len(CONV_ENTRIES)),
                         ids=[f"{e}-s{s}-{'-'.join(sorted(k))}" for e, s, k in CONV_ENTRIES])
@pytest.mark.parametrize("level", E.CONV_LEVELS, ids=[lv[0] for lv in E.CONV_LEVELS])
def test_conv_levels(ops, level, j, selector):
    """Every entry point at SDXL's latent levels (1024^2 and the 1216 x 832 bucket), odd H and W, B >= 3; dense
    integer weights, and selector weights whose picks visit every tap and both ends of every 64-channel block of every
    source (tap addressing, halo zeros, stride-2 parity maps, element for element)."""
    name, B, H, W, Cin, Cout = level
    entry, stride, kw = CONV_ENTRIES[j]
    conv_case(ops, entry, stride, kw, B, H, W, Cin, Cout, seed=3 * j + len(name), selector=selector)


@pytest.mark.parametrize("selector", [False, True])
@pytest.mark.parametrize("bw", sorted(E.BW_SHAPES, reverse=True))
def test_conv_every_spatial_tile(ops, bw, selector):
    Ho, Wo = E.BW_SHAPES[bw]
    assert E.pick_bw(Ho, Wo) == bw
    conv_case(ops, "conv", 1, dict(bias=True, rowbias=True, residual=True), 3, Ho, Wo, 128, 96, seed=bw,
              selector=selector)
    conv_case(ops, "down", 2, dict(bias=True), 3, 2 * Ho, 2 * Wo, 64, 64, seed=bw + 1, selector=selector)


@pytest.mark.parametrize("bn,B,H,W,Cin,Cout", E.conv_tile_cases())
def test_conv_forced_tiles(ops, bn, B, H, W, Cin, Cout):
    """Every forced tile width at < 1, 1-2 and >= 3 tiles per CTA, stride 1 and the down-sampling conv."""
    conv_case(ops, "conv", 1, dict(bias=True, residual=True), B, H, W, Cin, Cout, seed=bn + H, tile_n=bn)
    conv_case(ops, "down", 2, dict(bias=True), B, 2 * H, W, Cin, Cout, seed=bn + H + 1, tile_n=bn)


@pytest.mark.parametrize("cat", [False, True])
@pytest.mark.parametrize("B,H,W", [(2, 128, 128), (3, 37, 23), (2, 152, 104)])
def test_conv_in_im2col_gemm(ops, cat, B, H, W):
    """conv_in: ih_im2col3x3_nchw[_cat]_f16 patch matrix (k = c * 9 + tap) and the tensor-core GEMM, against the fp64
    convolution, bit for bit (4 latent channels, or latents | mask | masked-image latents)."""
    C0, C1 = (4, 5) if cat else (4, 0)
    C = C0 + C1
    kpad = 64 if C * 9 <= 64 else 128
    x = E.conv_input(B, H, W, C, B + H, "cuda")            # NHWC integers, then NCHW views for im2col
    xn = x.permute(0, 3, 1, 2).contiguous()
    w9 = E.dense(320, 9 * C, H, 1, "cuda")                    # [Cout, c * 9 + tap]
    bias = E.vec(320, -3, 3, W, "cuda")
    wk = torch.zeros(320, kpad, dtype=torch.float16, device="cuda")
    wk[:, :9 * C] = w9
    a = ops.im2col3x3_nchw_cat(xn[:, :C0].contiguous(), xn[:, C0:].contiguous(), kpad) if cat \
        else ops.im2col3x3_nchw(xn, kpad)
    out = ops.linear(a, wk, bias)
    # the same weight tap-major for conv_ref: [Cout, tap * C + c]
    w_tap = w9.view(320, C, 9).transpose(1, 2).reshape(320, 9 * C)
    ref = E.conv_ref(x, w_tap, bias=bias)
    assert float(ref.abs().max()) <= 2048
    assert E.check_bits(out.view(B, H, W, 320), ref) == 0, E.first_mismatch(out, ref.reshape(-1, 320))
