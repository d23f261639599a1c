"""CPU self-test of tests/exact_gemm.py: the builders' exactness claims, the coverage the GPU cases claim (every tile
at every ring-position class, every spatial tile width, every forced tile at every tiles-per-CTA class, every seam of
the sparse and selector weights), and that every simulated kernel defect fails its case's bar -- at >= 1 element for
bitwise cases, by >= 4x for the 1-ulp cases."""
import itertools

import pytest
import torch

import exact_gemm as E
from fp16_ulps import ulp16

# ---------------------------------------------------------------------------------------------------------------------
# exactness
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [8, 64, 200, 1024])
def test_fp32_sums_in_any_order_equal_fp64(chunk):
    """The premise: fp32 accumulation of the integer products in any chunking and order is exact."""
    M, N, K = 96, 80, 11520
    a, w = E.conv_input(1, 1, M, K, 5)[0, 0], E.conv_weight(N, K, 6)
    want = a.double() @ w.double().t()
    acc = torch.zeros(M, N, dtype=torch.float32)
    starts = list(range(0, K, chunk))
    for s in (starts[::-1] if chunk % 3 else starts):
        acc = acc + a[:, s:s + chunk].float() @ w[:, s:s + chunk].float().t()
    assert torch.equal(acc.double(), want)
    assert float(want.abs().max()) <= 2048


def _gelu_f32(x):
    """gelu_erf_f of ptx.cuh in float32 (erf_as: A&S 7.1.26 with ex2)."""
    x = x.float()
    ax = (x * 0.70710678118654752).abs()
    t = 1.0 / (0.3275911 * ax + 1.0)
    poly = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t
    e = torch.exp2(-ax * ax * 1.4426950408889634)
    r = torch.copysign(1.0 - poly * e, x)
    return (0.5 * x) * (1.0 + r)


def test_geglu_gates_saturate_erf_as():
    """|g| >= 8: erf_as is exactly +-1 in fp32, so gelu(g) is g or 0 and value * gelu(gate) is exact."""
    g = torch.arange(8, 2049, dtype=torch.float32)
    g = torch.cat([g, -g, g + 0.5, -g - 0.25])
    y = _gelu_f32(g)
    assert torch.equal(y, torch.where(g > 0, g, torch.zeros_like(g)))
    assert not torch.equal(_gelu_f32(torch.tensor([7.0, -3.0])), torch.tensor([7.0, 0.0]))   # not below


def _small_cases():
    """Every GPU GEMM case small enough to build here (and shrunk versions of the rest)."""
    out = []
    for i, (name, kw) in enumerate(E.PLAIN_EPILOGUES):
        for bn in E.PLAIN_STAGES:
            out.append((f"plain{bn}-{name}", E.epilogue_shape(False, bn, i), dict(kw)))
    for i, (name, kw) in enumerate(E.GEGLU_EPILOGUES):
        for bn in E.GEGLU_STAGES:
            out.append((f"geglu{bn}-{name}", E.epilogue_shape(True, bn, i), dict(kw, geglu=True, bias=True)))
    for i, (name, kw) in enumerate(E.SCALED_EPILOGUES):
        M, N, K = E.scaled_shape(128)
        out.append((f"scaled-{name}", (min(M, 777), N, K, 0), dict(kw)))
    for name, M, N, K, kw in E.SDXL_AUTO:
        kw = dict(kw, bias=True) if kw.get("geglu") else dict(kw)
        out.append((name, (min(M, 300), N, K, 4096 if kw.get("rowbias") else 0), kw))
    return out


@pytest.mark.parametrize("name,shape,kw", _small_cases(), ids=[c[0] for c in _small_cases()])
def test_gpu_case_bounds_and_bar(name, shape, kw):
    """The builders' claims on every GPU case: products and partial sums below 2^24, |y| <= 2048 where bitwise, GEGLU
    gates at |g| >= 8, activations in their window; fp16 of the exact result passes its own bar; a +-1 error of any
    accumulator costs >= 4 bars of a 1-ulp case."""
    M, N, K, rpg = shape
    c = E.gemm_case(M, N, K, seed=len(name), rows_per_group=rpg, **kw)
    ref, pre = E.gemm_ref(c)
    E.gemm_check_bounds(c, ref, pre)
    bad, r = E.gemm_bar(ref.half(), c, ref)
    assert bad == 0 or (bad is None and r <= 0.5 + 2 ** -10)
    if c["stats"]:
        assert E.stats_bad(E.stats_model(ref.half(), 64), ref.half()) == 0
    if not E.gemm_exact(c) and not c["geglu"]:
        # +-1 on the accumulator: pre moves by the accumulator's scale (alpha, or alpha * rstd)
        if c["act"] is not None:
            f = E.ACTS[c["act"]]
            step = c["alpha"]
            lo = (f(pre - step) - f(pre)).abs()
            hi = (f(pre + step) - f(pre)).abs()
        else:
            st = c["ln_stats"].double().sum(0)
            mean = st[:, 0] / K
            rstd = 1 / torch.sqrt((st[:, 1] / K - mean * mean).clamp_min(0) + c["eps"])
            lo = hi = rstd[:, None].expand_as(ref)
        bar = ulp16(ref) + c["slack"]
        assert float((torch.minimum(lo, hi) / bar).min()) >= 4


# ---------------------------------------------------------------------------------------------------------------------
# coverage
# ---------------------------------------------------------------------------------------------------------------------
def test_ring_cases_cover_every_instantiation_and_ring_class():
    seen = {}
    for geglu, bn, st, kb, per_cta, tail in E.ring_cases():
        M, N, K = E.ring_shape(geglu, bn, kb, per_cta, tail)
        bn_out = bn // 2 if geglu else bn
        tiles = -(-M // 128) * -(-(N // 2 if geglu else N) // bn_out)
        pos = "1" if kb == 1 else {st - 1: "S-1", st: "S", st + 1: "S+1"}.get(kb, "coprime")
        if pos == "coprime":
            assert all(kb % d for d in range(2, st + 1) if st % d == 0)
        assert -(-K // 64) == kb
        seen.setdefault((geglu, bn), set()).add((pos, E.ring_class(tiles)))
        seen.setdefault(("tails", geglu, bn), set()).add(K % 64)
    for geglu, table in ((False, E.PLAIN_STAGES), (True, E.GEGLU_STAGES)):
        for bn in table:
            want = set(itertools.product(["1", "S-1", "S", "S+1", "coprime"], ["<1", "1-2", ">=3"]))
            assert seen[(geglu, bn)] == want, (geglu, bn, want - seen[(geglu, bn)])
            assert seen[("tails", geglu, bn)] >= {0, 8, 56}


def test_epilogue_cases_cover_every_flag_on_every_tile():
    flags = set()
    for _, kw in E.PLAIN_EPILOGUES + E.SCALED_EPILOGUES:
        flags |= {k if k != "act" else v for k, v in kw.items() if v is not None and v is not False}
    assert flags >= {"bias", "rowbias", "residual", "silu", "gelu", "quick_gelu", "ln", "stats", "alpha", "relu"}
    assert {k for _, kw in E.GEGLU_EPILOGUES for k in kw} >= {"rowbias", "residual", "ln", "stats"}
    for bn in E.SCALED_TILES:
        M, N, K = E.scaled_shape(bn)
        m_tiles = -(-M // 128)
        assert E.pick_bn(m_tiles, N, -(-K // 64), True) == bn
    for bn in E.PLAIN_STAGES:   # rows_per_group seams inside tiles, not dividing M; K tails 8 / 56
        tails = {E.epilogue_shape(False, bn, i)[2] % 64 for i in range(3)}
        M, N, K, rpg = E.epilogue_shape(False, bn, 0)
        assert M % rpg and rpg % 128 and tails == {0, 8, 56}


def test_every_spatial_tile_and_forced_tile_is_reached():
    assert {E.pick_bw(ho, wo) for ho, wo in E.BW_SHAPES.values()} == {128, 64, 32, 16, 8, 4, 2, 1}
    for bw, (ho, wo) in E.BW_SHAPES.items():
        assert E.pick_bw(ho, wo) == bw and (ho % (128 // bw) or wo % bw or bw == 1)
    classes = {}
    for bn, B, H, W, Cin, Cout in E.conv_tile_cases():
        classes.setdefault(bn, set()).add(E.ring_class(E.conv_tiles(B, H, W, Cout, bn)))
    assert classes == {bn: {"<1", "1-2", ">=3"} for bn in E.FORCED_TILES}
    for _, B, H, W, _, _ in E.CONV_LEVELS:
        assert B >= 3 or (H, W) == (128, 128)
    assert {(H, W) for _, _, H, W, _, _ in E.CONV_LEVELS} >= {(152, 104), (76, 52), (38, 26), (37, 23)}


def test_sparse_rows_visit_every_seam():
    for K in (8, 56, 328, 1280, 11520):
        w = E.sparse_rows(64, K, 16, 3)
        seams = E.seam_cols(K)
        assert bool((w[:, seams] != 0).any(0).all()), K
        assert float(w.double().abs().sum(1).max()) <= 16


@pytest.mark.parametrize("Cin,sc", [(64, ()), (320, (320, 128)), (1280, (1280,))])
def test_selector_weights_visit_every_tap_and_channel_block_end(Cin, sc):
    w, targets = E.selector_weight(Cin if Cin < 1280 else 1280, Cin, sc, 1)
    nz = (w != 0).any(0).nonzero().flatten().tolist()
    assert targets <= set(nz)
    assert len(targets) == 9 * 2 * (Cin // 64) + sum(2 * (c // 64) for c in sc)


# ---------------------------------------------------------------------------------------------------------------------
# defects
# ---------------------------------------------------------------------------------------------------------------------
def _fails(out, c, ref, name):
    bad, r = E.gemm_bar(out, c, ref)
    if bad is not None:
        print(f"[defect] {name}: {bad} elements differ")
        return bad >= 1
    print(f"[defect] {name}: fails by {r:.1f}x the 1-ulp bar")
    return r >= 4


GEMM_DEFECTS = [
    # (defect, case kwargs, stages)
    ("drop", dict(bias=True), None),
    ("double", dict(bias=True), None),
    ("stale", dict(bias=True), 4),
    ("other_tile", dict(bias=True), None),
    ("k_tail", dict(bias=True), None),
    ("geglu_swap", dict(geglu=True, bias=True), None),
    ("gate_group", dict(geglu=True, bias=True), None),
    ("rowbias_group", dict(rowbias=True, bias=True), None),
    ("residual_row", dict(residual=True), None),
    ("alpha_bias", dict(alpha=0.25, bias=True), None),
    ("ln_inv_c", dict(ln=True, bias=True), None),
    ("ln_row", dict(ln=True, bias=True), None),
    ("ln_inv_c", dict(ln=True, geglu=True, bias=True), None),
    ("ln_inv_c", dict(ln=True), None),
    ("drop", dict(act="gelu", bias=True), None),
    ("double", dict(act="silu"), None),
    ("other_tile", dict(act="quick_gelu", rowbias=True), None),
    ("drop", dict(ln=True, geglu=True, bias=True), None),
]


@pytest.mark.parametrize("defect,kw,stages", GEMM_DEFECTS, ids=[f"{d}-{'-'.join(k)}" for d, k, _ in GEMM_DEFECTS])
@pytest.mark.parametrize("K", [328, 1280])
def test_gemm_defect_fails(defect, kw, stages, K):
    M, N = 300, 256
    c = E.gemm_case(M, N, K, seed=5, rows_per_group=100, **kw)
    ref, _ = E.gemm_ref(c)
    bad, _ = E.gemm_ref(c, defect=defect, stages=stages, kb=None if defect != "stale" else 5)
    assert _fails(bad.half(), c, ref, f"{defect} {sorted(kw)} K={K}")


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("defect", ["slot_missing", "wrong_slot", "lost_carry"])
def test_stats_defect_fails(bn, defect):
    if defect == "lost_carry" and bn != 160:
        pytest.skip("the carry exists in the 160-column tile only")
    c = E.gemm_case(300, 640, 328, seed=9, stats=True, bias=True)
    ref, _ = E.gemm_ref(c)
    out = ref.half()
    assert E.stats_bad(E.stats_model(out, bn), out) == 0
    bad = E.stats_bad(E.stats_model(out, bn, defect), out)
    print(f"[defect] stats {defect} (tile {bn}): {bad} rows differ")
    assert bad >= 1


CONV_DEFECTS = [
    ("tap_x+", dict(), 1), ("tap_x-", dict(), 1), ("tap_y+", dict(), 1), ("tap_y-", dict(), 1),
    ("wrap", dict(), 1), ("parity", dict(), 2), ("pad_side", dict(), 2), ("pad_side", dict(pad="br"), 2),
    ("sc_swap", dict(sources=2), 1), ("sc_drop", dict(sources=2), 1), ("sc_drop", dict(sources=1), 1),
    ("rowbias_group", dict(rowbias=True), 1), ("residual_row", dict(residual=True), 1),
    ("alpha_bias", dict(alpha=0.5), 1),
]


@pytest.mark.parametrize("selector", [False, True])
@pytest.mark.parametrize("defect,kw,stride", CONV_DEFECTS, ids=[f"{d}-{'-'.join(k)}-s{s}" for d, k, s in CONV_DEFECTS])
def test_conv_defect_fails(defect, kw, stride, selector):
    B, H, W, Cin, Cout = 3, 10, 7 * stride, 64, 64
    x = E.conv_input(B, H, W, Cin, 2)
    sc = [E.conv_input(B, H, W, 64, 3 + i) for i in range(kw.get("sources", 0))]
    if selector:
        w, _ = E.selector_weight(Cout, Cin, [s.shape[-1] for s in sc], 4)
    else:
        w = E.conv_weight(Cout, 9 * Cin + 64 * len(sc), 4)
    extra = dict(bias=E.vec(Cout, -3, 3, 5), alpha=kw.get("alpha", 1.0), stride=stride, pad=kw.get("pad", "all"),
                 shortcut=sc)
    if kw.get("rowbias"):
        extra["rowbias"] = E.ints(B, Cout, -3, 3, 6).half()
    if kw.get("residual"):
        extra["residual"] = E.ints(B * (H // stride) * (W // stride), Cout, -4, 4, 7).half().view(
            B, H // stride, W // stride, Cout)
    ref = E.conv_ref(x, w, **extra)
    E.conv_check_bounds(x, w, ref, sc)
    assert E.check_bits(ref.half(), ref) == 0
    bad = E.check_bits(E.conv_ref(x, w, defect=defect, **extra).half(), ref)
    print(f"[defect] conv {defect} {sorted(kw)} stride {stride} selector={selector}: {bad} elements differ")
    assert bad >= 1
