"""GPU tests of the ping-pong GEMM kernel (gemm_pp_f16_kernel, forced with tile_n = TILE_PINGPONG): its outputs must be
bitwise equal to gemm_f16_kernel's -- the 256-row tile for GEGLU, the plain tiles for q|k|v -- because the automatic
choice switches between the two kernels by shape."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    torch.backends.cuda.matmul.allow_tf32 = False
    from imagharmony_b200 import ops as _ops
    return _ops


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def ln_stats(m, k, seed=0):
    """Row statistics [ceil(K/64), M, 2] as a producing GEMM writes them: per slab (sum, sum of squares)."""
    g = torch.Generator(device="cpu").manual_seed(seed + m + k)
    s = torch.randn(((k + 63) // 64, m, 2), generator=g)
    s[..., 1] = s[..., 1].abs() * 8 + 64.0
    return s.cuda()


def launch(ops, x, w, b, geglu, ln, tile_n, out=None):
    return ops.linear(x, w, b, geglu=geglu, ln=None if ln is None else (ln, 1e-5), tile_n=tile_n, out=out)


def old_tile(geglu):
    return 256 if geglu else 128


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def check_equal(ops, m, n, k, geglu, bias=True, ln=True, seed=0):
    x, w = rnd(m, k, seed=seed), rnd(n, k, scale=k ** -0.5, seed=seed + 1)
    b = rnd(n, scale=0.5, seed=seed + 2) if bias else None
    st = ln_stats(m, k, seed) if ln else None
    pp = launch(ops, x, w, b, geglu, st, ops.TILE_PINGPONG)
    ref = launch(ops, x, w, b, geglu, st, old_tile(geglu))
    assert torch.isfinite(ref).all()
    assert torch.equal(pp, ref), (m, n, k, geglu, bias, ln, (pp.float() - ref.float()).abs().max().item())
    if not ln:   # and against fp32: the kernel computes what it should, not only what the old one does
        y = x.float() @ w.float().t() + (0 if b is None else b.float())
        want = y[:, :n // 2] * F.gelu(y[:, n // 2:]) if geglu else y
        torch.testing.assert_close(pp.float(), want, rtol=2e-3, atol=2e-3)
    return pp


# the LayerNorm-folded q|k|v (N = 3C) and GEGLU (N = 8C) launches of the SDXL base UNet (C 640 / 1280) and refiner
# (C 768 / 1536) at 512^2 - 1024^2, M = 2 * images * tokens
UNET_SHAPES = [(2 * 1 * 1024, 1280), (2 * 1 * 4096, 640), (2 * 1 * 256, 1280), (2 * 4 * 1024, 640),
               (2 * 1 * 1024, 1536), (2 * 1 * 4096, 768), (2 * 4 * 576, 1536)]


@pytest.mark.parametrize("geglu", [False, True])
@pytest.mark.parametrize("m,c", UNET_SHAPES)
def test_unet_shapes(ops, m, c, geglu):
    check_equal(ops, m, 8 * c if geglu else 3 * c, c, geglu)


@pytest.mark.parametrize("geglu", [False, True])
@pytest.mark.parametrize("bias,ln", [(False, False), (True, False), (False, True), (True, True)])
def test_bias_and_ln(ops, geglu, bias, ln):
    check_equal(ops, 3000, 2560, 640, geglu, bias=bias, ln=ln)


@pytest.mark.parametrize("geglu", [False, True])
@pytest.mark.parametrize("m,n_out,k", [
    (1000, 1000, 640),    # ragged M (1000 = 7 * 128 + 104) and ragged N (not a multiple of 128 / 64 outputs)
    (129, 200, 320),      # one row past a tile; N 200 ends inside a 64-column slab
    (777, 328, 64),       # K = 64: one k-block per tile
    (500, 264, 200),      # K not a multiple of 64 (TMA zero fill of the last k-block)
    (128, 128, 1280),     # one tile (GEGLU: two) -- the second MMA warpgroup of a CTA may have nothing to do
    (128, 64, 640),       # exactly one tile in both modes
])
def test_edges(ops, m, n_out, k, geglu):
    check_equal(ops, m, 2 * n_out if geglu else n_out, k, geglu, ln=k % 64 == 0, seed=3)


@pytest.mark.parametrize("geglu", [False, True])
@pytest.mark.parametrize("per_cta", [0.5, 1, 2, 3, 5])
def test_tiles_per_cta(ops, geglu, per_cta):
    """Tile counts below the SM count, equal to it, and two / three / five per CTA (odd counts leave the first
    warpgroup one tile more than the second)."""
    tiles = max(1, int(per_cta * sms()))
    n_out = 128 * 8
    per_row = n_out // (64 if geglu else 128)
    m = 128 * (-(-tiles // per_row))
    check_equal(ops, m, 2 * n_out if geglu else n_out, 640, geglu, seed=5)


@pytest.mark.parametrize("geglu", [False, True])
def test_strided_rows(ops, geglu):
    """lda and ldo larger than the row: A is a column slice, the output a column slice of a wider buffer."""
    m, k, n = 1500, 640, 1024
    big = rnd(m, k + 192, seed=7)
    x = big[:, 64:64 + k]
    w, b = rnd(n, k, scale=k ** -0.5, seed=8), rnd(n, seed=9)
    st = ln_stats(m, k, 7)
    n_out = n // 2 if geglu else n
    buf = torch.full((m, n_out + 136), 7.0, dtype=torch.float16, device="cuda")
    out = buf[:, 72:72 + n_out]
    launch(ops, x, w, b, geglu, st, ops.TILE_PINGPONG, out=out)
    ref = launch(ops, x.contiguous(), w, b, geglu, st, old_tile(geglu))
    assert torch.equal(out, ref)
    assert (buf[:, :72] == 7.0).all() and (buf[:, 72 + n_out:] == 7.0).all()


def test_unsupported_epilogue_refused(ops):
    from imagharmony_b200._lib import IHError
    x, w = rnd(256, 320), rnd(384, 320, scale=320 ** -0.5)
    with pytest.raises(IHError):
        ops.linear(x, w, residual=rnd(256, 384), tile_n=ops.TILE_PINGPONG)
    with pytest.raises(IHError):
        ops.linear(x, w, silu=True, tile_n=ops.TILE_PINGPONG)


def kernels_run(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "gemm" in e.name}


def test_auto_picks_pingpong_at_unet_geglu(ops):
    """The automatic choice runs the ping-pong kernel for the 1024^2 level-2 GEGLU launch (the cost model in gemm.cu,
    fitted to tools/ab_probe.py pp: DESIGN section 3), and the old kernel for the explicit 256-row tile."""
    m, c = 2048, 1280
    x, w, b = rnd(m, c), rnd(8 * c, c, scale=c ** -0.5), rnd(8 * c)
    st = ln_stats(m, c)
    names = kernels_run(lambda: launch(ops, x, w, b, True, st, 0))
    assert any("gemm_pp_f16_kernel" in n for n in names), names
    names = kernels_run(lambda: launch(ops, x, w, b, True, st, 256))
    assert not any("gemm_pp_f16_kernel" in n for n in names), names


def test_dependent_launch_and_graph_replay(ops):
    """A ping-pong launch followed directly by launches that read its output (programmatic dependent launch), eager
    and replayed as a CUDA graph, gives the old kernel's results bit for bit."""
    m, c = 2048, 640
    h = rnd(m, c, seed=11)
    st = ln_stats(m, c, 11)
    w1, b1 = rnd(8 * c, c, scale=c ** -0.5, seed=12), rnd(8 * c, seed=13)
    wq, bq = rnd(3 * c, c, scale=c ** -0.5, seed=14), rnd(3 * c, seed=15)
    w2, b2 = rnd(c, 4 * c, scale=(4 * c) ** -0.5, seed=16), rnd(c, seed=17)

    def chain(tile_geglu, tile_plain):
        g = launch(ops, h, w1, b1, True, st, tile_geglu)
        o = ops.linear(g, w2, b2, residual=h)              # reads g right behind the GEGLU launch
        q = launch(ops, o, wq, bq, False, None, tile_plain)
        return g, o, launch(ops, q[:, :c], wq, None, False, None, tile_plain)

    ref = [t.clone() for t in chain(256, 128)]
    got = [t.clone() for t in chain(ops.TILE_PINGPONG, ops.TILE_PINGPONG)]
    for a, e in zip(got, ref):
        assert torch.equal(a, e)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain(ops.TILE_PINGPONG, ops.TILE_PINGPONG)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = chain(ops.TILE_PINGPONG, ops.TILE_PINGPONG)
    for _ in range(2):
        for t in outs:
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for a, e in zip(outs, ref):
            assert torch.equal(a, e)
