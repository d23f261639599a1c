"""GPU tests of the epilogue of gemm_f16_kernel across its tile widths: every plain tile (64 / 128 / 160 / 192 / 256
columns) and every GEGLU tile (128 / 192 / 256 B-tile rows), plain GEMM and implicit-GEMM conv, with every epilogue
operand.  The launches are sized so each CTA walks three or more tiles: staging is written by one tile's epilogue while
the previous tile's stores may still be reading it out, so a multi-round launch is where a missing wait shows."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PLAIN_TILES = [64, 128, 160, 192, 256]
GEGLU_TILES = [128, 192, 256]


@pytest.fixture(scope="module")
def ops():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from imagharmony_b200 import ops as _ops
    return _ops


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def check(out, ref, what, tol=2e-3):
    out, ref = out.float(), ref.float()
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs()
    bound = tol + tol * ref.abs() + ref.abs() * 2.0 ** -11     # one fp16 rounding of the fp32 reference
    frac = (err > bound).float().mean().item()
    assert frac == 0.0, f"{what}: {frac:.3e} of elements out of tolerance, max err {err.max().item():.3e}"


def rounds(m_rows, n_out, cols):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-m_rows // 128) * -(-n_out // cols)
    return -(-tiles // sms)


# M = 8000: 63 row tiles, the last one 64 rows short; N = 1480 is no multiple of any tile width
M, N, K = 8000, 1480, 640


@pytest.mark.parametrize("bn", PLAIN_TILES)
@pytest.mark.parametrize("epi", ["none", "bias", "bias+residual", "rowbias+silu", "gelu", "quick_gelu"])
def test_plain_tiles(ops, bn, epi):
    assert rounds(M, N, bn) >= 3
    x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N, scale=0.5)
    res, rb = rnd(M, N, seed=3), rnd(2, N, seed=5)
    acc = x.float() @ w.float().t()
    kw = {}
    bias = None if epi == "none" else b
    ref = acc if bias is None else acc + b.float()
    if epi == "bias+residual":
        kw["residual"], ref = res, ref + res.float()
    elif epi == "rowbias+silu":
        kw.update(rowbias=rb, rows_per_group=M // 2, silu=True)
        ref = F.silu(ref + rb.float().repeat_interleave(M // 2, dim=0))
    elif epi == "gelu":
        kw["gelu"], ref = True, F.gelu(ref)
    elif epi == "quick_gelu":
        kw["quick_gelu"], ref = True, ref * torch.sigmoid(1.702 * ref)
    out = ops.linear(x, w, bias, tile_n=bn, **kw)
    check(out, ref, f"gemm bn{bn} {epi}")
    # the k order of the accumulation does not depend on the tile width
    assert torch.equal(out, ops.linear(x, w, bias, tile_n=128, **kw))


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("m,n", [(8000, 1480), (2048, 1280), (300, 72)])
def test_alpha_relu(ops, m, n, relu):
    """alpha and ReLU take the library's tile choice: relu(alpha * acc + bias + residual) / alpha * acc + bias + residual."""
    x, w, b, res = rnd(m, K), rnd(n, K, scale=K ** -0.5), rnd(n), rnd(m, n, seed=7)
    ref = 0.25 * (x.float() @ w.float().t()) + b.float() + res.float()
    if relu:
        ref = torch.relu(ref)
    check(ops.linear(x, w, b, residual=res, alpha=0.25, relu=relu), ref, f"alpha relu={relu} {m}x{n}")


@pytest.mark.parametrize("bn", [64, 128, 160, 192, 256])
def test_stats_out(ops, bn):
    """Row statistics: every slot written once, the slot sums are the rows' sums of the stored fp16 values."""
    m, n = 8000, 1280
    assert rounds(m, n, bn) >= 3
    x, w, b, res = rnd(m, K), rnd(n, K, scale=K ** -0.5), rnd(n), rnd(m, n, seed=3)
    stats = torch.full((n // 64, m, 2), float("nan"), dtype=torch.float32, device="cuda")
    h = ops.linear(x, w, b, residual=res, stats_out=stats, tile_n=bn)
    check(h, x.float() @ w.float().t() + b.float() + res.float(), f"stats bn{bn}")
    assert torch.isfinite(stats).all()
    hf = h.float()
    s = stats.sum(dim=0)
    torch.testing.assert_close(s[:, 0], hf.sum(dim=1), rtol=1e-5, atol=1e-3)
    torch.testing.assert_close(s[:, 1], (hf * hf).sum(dim=1), rtol=1e-5, atol=1e-3)
    assert torch.equal(h, ops.linear(x, w, b, residual=res, tile_n=128))


def geglu_ref(x, w, b):
    y = x.float() @ w.float().t() + b.float()
    f = y.shape[1] // 2
    return y[:, :f] * F.gelu(y[:, f:])


@pytest.mark.parametrize("bn", GEGLU_TILES)
@pytest.mark.parametrize("m,n_out,k", [(8000, 1000, 640), (2048, 5120, 1280), (300, 40, 200)])
def test_geglu_tiles(ops, bn, m, n_out, k):
    """Every GEGLU tile matches the reference and, bit for bit, the 256-row tile (GEGLU writes no statistics and
    the k order does not depend on the tile)."""
    x, w, b = rnd(m, k), rnd(2 * n_out, k, scale=k ** -0.5), rnd(2 * n_out, scale=0.5)
    out = ops.linear(x, w, b, geglu=True, tile_n=bn)
    check(out, geglu_ref(x, w, b), f"geglu bn{bn} {m}x{n_out}x{k}")
    assert torch.equal(out, ops.linear(x, w, b, geglu=True, tile_n=256))
    assert torch.equal(out, ops.linear(x, w, b, geglu=True))


def test_geglu_192_refuses_stats(ops):
    from imagharmony_b200._lib import IHError
    m, n_out = 512, 256
    x, w = rnd(m, K), rnd(2 * n_out, K, scale=K ** -0.5)
    stats = torch.full((n_out // 64, m, 2), float("nan"), dtype=torch.float32, device="cuda")
    with pytest.raises(IHError):
        ops.linear(x, w, geglu=True, stats_out=stats, tile_n=192)
    g = ops.linear(x, w, geglu=True, stats_out=stats)          # the library's choice avoids the 96-output tile
    torch.testing.assert_close(stats.sum(dim=0)[:, 0], g.float().sum(dim=1), rtol=1e-5, atol=1e-3)


def ln_producer(ops, m, c):
    a, wp, bp = rnd(m, c, seed=31), rnd(c, c, scale=c ** -0.5, seed=32), rnd(c, seed=33)
    res = rnd(m, c, seed=34) * 2 + 0.5
    stats = torch.full((c // 64, m, 2), float("nan"), dtype=torch.float32, device="cuda")
    h = ops.linear(a, wp, bp, residual=res, stats_out=stats)
    gamma = (1 + 0.2 * rnd(c, seed=35).float()).half()
    beta = (0.1 * rnd(c, seed=36).float()).half()
    return h, stats, gamma, beta


@pytest.mark.parametrize("geglu,bn", [(False, t) for t in PLAIN_TILES] + [(True, t) for t in GEGLU_TILES])
def test_layernorm_fold_rounds(ops, geglu, bn):
    """Folded LayerNorm consumers (q|k|v, GEGLU): the multi-round launch matches the explicit LayerNorm, and each row
    equals the same row of a launch over a few rows only (one round)."""
    m, c = 8000, 640
    n = 4 * c if geglu else 3 * c
    h, stats, gamma, beta = ln_producer(ops, m, c)
    w, b = rnd(n, c, scale=c ** -0.5, seed=37), rnd(n, scale=0.25, seed=38)
    w_c, cvec = ops.fold_layernorm(w, b, gamma, beta)
    out = ops.linear(h, w_c, cvec, geglu=geglu, ln=(stats, 1e-5), tile_n=bn)
    assert rounds(m, out.shape[1], bn // 2 if geglu else bn) >= 3
    ln = F.layer_norm(h.float(), (c,), gamma.float(), beta.float(), 1e-5)
    y = ln @ w.float().t() + b.float()
    ref = y[:, :n // 2] * F.gelu(y[:, n // 2:]) if geglu else y
    check(out, ref, f"ln-fold geglu={geglu} bn{bn}", tol=1e-2)
    for r0, r1 in [(0, 128), (1024, 1280), (m - 200, m)]:
        part = ops.linear(h[r0:r1], w_c, cvec, geglu=geglu, ln=(stats[:, r0:r1].contiguous(), 1e-5), tile_n=bn)
        assert rounds(r1 - r0, out.shape[1], bn // 2 if geglu else bn) == 1
        assert torch.equal(part, out[r0:r1]), (r0, r1)


def conv_ref(x, w_packed, bias, stride=1):
    cout, cin = w_packed.shape[0], x.shape[-1]
    w4 = w_packed[:, :9 * cin].float().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    return F.conv2d(x.float().permute(0, 3, 1, 2), w4, bias.float(), stride=stride, padding=1).permute(0, 2, 3, 1)


@pytest.mark.parametrize("bn", PLAIN_TILES)
@pytest.mark.parametrize("stride,cout,epi", [(1, 640, "bias"), (1, 200, "residual"), (1, 640, "rowbias"),
                                             (2, 640, "bias")])
def test_conv_tiles(ops, bn, stride, cout, epi):
    bsz, hw, cin = 2, 64 if stride == 1 else 128, 640
    x, w, b = rnd(bsz, hw, hw, cin), rnd(cout, 9 * cin, scale=(9 * cin) ** -0.5), rnd(cout)
    ho = hw // stride
    assert cout != 640 or rounds(bsz * ho * ho, cout, bn) >= 2
    ref = conv_ref(x, w, b, stride)
    kw = {}
    if epi == "residual":
        kw["residual"] = rnd(bsz, ho, ho, cout, seed=4)
        ref = ref + kw["residual"].float()
    elif epi == "rowbias":
        kw["rowbias"] = rnd(bsz, cout, seed=6)
        ref = ref + kw["rowbias"].float()[:, None, None, :]
    out = ops.conv3x3(x, w, b, stride=stride, tile_n=bn, **kw)
    check(out, ref, f"conv bn{bn} s{stride} {epi}", tol=4e-3)
    assert torch.equal(out, ops.conv3x3(x, w, b, stride=stride, tile_n=128, **kw))


@pytest.mark.parametrize("hw,c", [(64, 640), (32, 1280)])
def test_conv_shortcut_taps(ops, hw, c):
    """Fused 1x1 shortcut over two sources (the up-block ResBlock: hidden state and skip), library's tile choice."""
    bsz = 2
    x, s0, s1 = rnd(bsz, hw, hw, c), rnd(bsz, hw, hw, c, seed=11), rnd(bsz, hw, hw, c // 2, seed=12)
    csc = c + c // 2
    w, b = rnd(c, 9 * c + csc, scale=(9 * c + csc) ** -0.5), rnd(c)
    out = ops.conv3x3(x, w, b, shortcut=(s0, s1))
    ref = conv_ref(x, w, b) + torch.cat([s0, s1], dim=-1).float() @ w[:, 9 * c:].float().t()
    check(out, ref, f"conv+shortcut {hw}^2 C{c}", tol=4e-3)


def test_graph_replay_bit_identical(ops):
    """A feed-forward chain (statistics producer -> LayerNorm-folded GEGLU -> FF-out with residual and statistics) on
    the library's tile choices, replayed as a CUDA graph, reproduces the eager results bit for bit."""
    m, c = 2048, 1280
    h, stats, gamma, beta = ln_producer(ops, m, c)
    w1, b1 = rnd(8 * c, c, scale=c ** -0.5, seed=41), rnd(8 * c, seed=42)
    w_c, cvec = ops.fold_layernorm(w1, b1, gamma, beta)
    w2, b2 = rnd(c, 4 * c, scale=(4 * c) ** -0.5, seed=43), rnd(c, seed=44)
    st2 = torch.empty((c // 64, m, 2), dtype=torch.float32, device="cuda")

    def chain():
        g = ops.linear(h, w_c, cvec, geglu=True, ln=(stats, 1e-5))
        return g, ops.linear(g, w2, b2, residual=h, stats_out=st2)

    g_e, o_e = (t.clone() for t in chain())
    st_e = st2.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_g, o_g = chain()
    for _ in range(2):
        st2.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(g_g, g_e) and torch.equal(o_g, o_e) and torch.equal(st2, st_e)
