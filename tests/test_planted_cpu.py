"""The planted-marker cases of test_planted_gpu.py keep their power to catch a broken kernel: for each family, at a
small but representative size, the fp16-rounded fp64 reference passes its bar with room to spare, and every simulated
bookkeeping defect (a marker dropped or counted twice, an element credited to the neighbouring image, row or group, a
padding key or column let in, the online-softmax rescale omitted, a KV part's combine weight wrong, a row chunk's
partial missing, the rescale std taken over the wrong image) fails it by at least DEFECT_MARGIN."""
import pytest
import torch

import planted as P

EXACT_MAX = 0.6          # an fp16 rounding of the exact result is at most half an ulp away
DEFECT_MARGIN = 4.0


def r16(t):
    return t.half().double()


def report(what, exact, defects):
    print(f"[planted {what}] exact {exact:.3f}  " + "  ".join(f"{k} {v:.1f}" for k, v in defects.items()))
    assert exact <= EXACT_MAX, (what, exact)
    weak = {k: v for k, v in defects.items() if not v >= DEFECT_MARGIN}
    assert not weak, (what, weak)


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,HW,C0,C1,groups,silu", [
    (2, 2048, 320, 0, 32, True),     # 32 markers per (image, group): the most any GPU case has
    (3, 256, 1280, 0, 160, False),
    (2, 100, 640, 0, 320, True),     # groups = C / 2
    (4, 7, 320, 0, 32, False),       # fewer rows than groups: several groups per marker row
    (2, 512, 1280, 640, 32, True),   # a group straddles the x0 | x1 seam
])
def test_groupnorm_planted_defects_fail(B, HW, C0, C1, groups, silu):
    eps = 1e-5
    C = C0 + C1
    gamma, beta = P.gn_params(C)
    cover = P.gn_cover_rows(B, HW, C)
    n_launch = P.gn_launches(B, HW, C, groups)
    _, rpb, _ = P.gn_plan(B, HW, C)
    cpg = C // groups
    exact, per_launch = 0.0, []
    for L in range(n_launch):
        mk = P.gn_markers(B, HW, C, groups, L, n_launch, cover, C0 if C1 else None)
        x = P.gn_build(B, HW, C, mk)
        s, q = P.gn_sums(x, groups)
        per_g = torch.zeros(B, groups)
        per_g.index_put_((mk[0], mk[2] // cpg), torch.ones(len(mk[0])), accumulate=True)
        assert per_g.min() >= 1 and per_g.max() <= P.GN_PER_GROUP, (per_g.min(), per_g.max())

        def rr(sums):
            return P.gn_check_ratio(r16(P.gn_reference(x, gamma, beta, groups, eps, silu, sums)[0]), x, gamma, beta,
                                    groups, eps, silu)

        def group_rr(b, g, ds, dq):
            """rr of a defect that moves only the sums of (image b, group g): that group's outputs, on their own."""
            cols = slice(g * cpg, (g + 1) * cpg)
            xs, ga, be = x[b:b + 1, :, cols], gamma[cols], beta[cols]
            sums = (s[b:b + 1, g:g + 1] + ds, q[b:b + 1, g:g + 1] + dq)
            return P.gn_check_ratio(r16(P.gn_reference(xs, ga, be, 1, eps, silu, sums)[0]), xs, ga, be, 1, eps, silu)
        exact = max(exact, rr(None))
        # every marker, by its (image, group, value): dropped, counted twice, credited to the next group
        d = {"drop": float("inf"), "double": float("inf"), "group": float("inf")}
        for b, g, v in sorted({(int(b), int(c) // cpg, float(v)) for b, c, v in zip(mk[0], mk[2], mk[3])}):
            d["drop"] = min(d["drop"], group_rr(b, g, -v, -v * v))
            d["double"] = min(d["double"], group_rr(b, g, v, v * v))
            d["group"] = min(d["group"], max(group_rr(b, g, -v, -v * v), group_rr(b, (g + 1) % groups, v, v * v)))
        xs = x.double().view(B, HW, groups, cpg)
        # image b + 1's first row counted in image b
        d["image"] = [rr((s + torch.nn.functional.pad(xs[1:, 0].sum(-1), (0, 0, 0, 1)),
                          q + torch.nn.functional.pad((xs[1:, 0] ** 2).sum(-1), (0, 0, 0, 1))))] if B > 1 else []
        # one row chunk's partial (two-kernel plan) missing, in each image
        chunks = []
        for b in range(B):
            for r0 in range(0, HW, rpb):
                part = xs[b, r0:r0 + rpb]
                s2, q2 = s.clone(), q.clone()
                s2[b] -= part.sum((0, 2))
                q2[b] -= (part ** 2).sum((0, 2))
                chunks.append(rr((s2, q2)))
        d["chunk"] = chunks
        per_launch.append(d)
    # a marker defect is caught in its own launch; a row defect in any launch where that row carries a marker
    defects = {k: min(d[k] for d in per_launch) for k in ("drop", "double", "group")}
    if B > 1:
        defects["image"] = max(d["image"][0] for d in per_launch)
    defects["chunk"] = min(max(d["chunk"][i] for d in per_launch) for i in range(len(per_launch[0]["chunk"])))
    report(f"groupnorm B{B} HW{HW} C{C0}+{C1} g{groups} silu{silu} x{n_launch}", exact, defects)


@pytest.mark.parametrize("B,HW,C0,C1,groups,silu,scale", P.GN_CASES)
def test_groupnorm_gpu_cases_mark_every_seam_channel(B, HW, C0, C1, groups, silu, scale):
    """Over the launches of every GPU case, every group's first and last channel, both ends of every 8-channel vector
    and both sides of the x0 | x1 seam carry a marker, and every cover row is a marker row."""
    C = C0 + C1
    cover = P.gn_cover_rows(B, HW, C)
    n = P.gn_launches(B, HW, C, groups)
    ch_seen = torch.zeros(C, dtype=torch.bool)
    row_seen = torch.zeros(B, HW, dtype=torch.bool)
    for L in range(n):
        b, r, c, _ = P.gn_markers(B, HW, C, groups, L, n, cover, C0 if C1 else None)
        ch_seen[c] = True
        row_seen[b, r] = True
    need = P.gn_seam_channels(C, groups, C0 if C1 else None)
    cpg = C // groups
    assert {0, cpg - 1, C - 1} <= set(need.tolist())
    if C1:
        assert {C0 - 1, C0} <= set(need.tolist())
    assert bool(ch_seen[need].all()), f"seam channels without a marker: {need[~ch_seen[need]].tolist()[:16]}"
    assert bool(row_seen[:, cover].all()), "cover rows without a marker"


def test_groupnorm_cover_rows_hold_every_plan_seam():
    """At the VAE's 1024^2 level the covered rows include both sides of every chunk boundary of both plans and of
    every multiple of 4R, the first and the last row, and the launches keep at most GN_PER_GROUP markers per group."""
    B, HW, C, groups = 1, 1 << 20, 128, 32
    cover = set(P.gn_cover_rows(B, HW, C).tolist())
    R, rpb, fused = P.gn_plan(B, HW, C)
    assert len(fused) > 100 and {0, HW - 1} <= cover
    for step in [4 * R, rpb] + fused:
        assert all(m - 1 in cover and m in cover for m in range(step, HW, step)), step
    n = P.gn_launches(B, HW, C, groups)
    mk = P.gn_markers(B, HW, C, groups, n - 1, n, torch.tensor(sorted(cover)))
    assert torch.bincount(mk[2] // (C // groups), minlength=groups).max() <= P.GN_PER_GROUP
    print(f"[planted groupnorm VAE 1024^2] {len(cover)} cover rows in {n} launches")


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
def _ln_stats(xs, w):
    C = xs.shape[-1]
    mean = (xs * w).sum(-1, keepdim=True) / C
    return mean, (w * (xs - mean) ** 2).sum(-1, keepdim=True) / C


@pytest.mark.parametrize("C", [8, 264, 2048, 8192])
def test_layernorm_planted_defects_fail(C):
    rows = P.ln_rows(C, 3)
    x = P.ln_build(rows, C)
    g, b = P.ln_params(C)
    xd = x.double()

    def rr(stats):
        ref, slack = P.ln_reference(x, g, b, 1e-5)
        return P.ratio(r16(P.ln_reference(x, g, b, 1e-5, stats)[0]), ref, 1.0, slack)
    exact = rr(None)
    d = {"drop": float("inf"), "double": float("inf"), "row": float("inf")}
    for r in range(min(rows - 1, 8)):
        for j in torch.nonzero(xd[r] != P.LN_OFFSET).flatten().tolist():
            for name, wv in (("drop", 0.0), ("double", 2.0)):
                w = torch.ones_like(xd)
                w[r, j] = wv
                d[name] = min(d[name], rr(_ln_stats(xd, w)))
        for j in torch.nonzero(xd[r + 1] != xd[r]).flatten().tolist()[:4]:
            xs = xd.clone()
            xs[r, j] = xd[r + 1, j]                # row r + 1's element in row r's statistics
            d["row"] = min(d["row"], rr(_ln_stats(xs, torch.ones_like(xd))))
    report(f"layernorm {rows}x{C}", exact, d)


# ---------------------------------------------------------------------------------------------------------------------
# masked row softmax
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols,valid", [(168, 1), (168, 9), (168, 167), (4096, 4095), (4096, 4096)])
def test_softmax_planted_defects_fail(cols, valid):
    rows = 12
    buf, x = P.smx_build(rows, cols, valid, cols + 64)
    ref = P.smx_reference(x, valid)
    d = {}
    if valid < cols:
        d["pad"] = P.ratio(r16(P.smx_reference(x, valid + 1)), ref)
    drop, dbl, row = [], [], []
    xd = x.double()
    for r in range(rows - 1):
        for j in torch.nonzero(xd[r, :valid] == P.SMX_TOP).flatten().tolist():
            xs = xd.clone()
            xs[r, j] = -float("inf")
            drop.append(P.ratio(r16(P.smx_reference(xs, valid)), ref))
            e = torch.exp(xd[r, :valid] - P.SMX_TOP)
            bad = ref.clone()
            bad[r, :valid] = e / (e.sum() + e[j])
            dbl.append(P.ratio(r16(bad), ref))
        nb = torch.nonzero((xd[r + 1, :valid] == P.SMX_TOP) & (xd[r, :valid] != P.SMX_TOP)).flatten().tolist()
        if nb:                                     # row r + 1's maximum in row r's sum
            e = torch.exp(xd[r, :valid] - P.SMX_TOP)
            bad = ref.clone()
            bad[r, :valid] = e / (e.sum() + 1.0)
            row.append(P.ratio(r16(bad), ref))
    d.update(drop=min(drop), double=min(dbl))
    if row:
        d["row"] = min(row)
    report(f"softmax {cols} valid {valid}", P.ratio(r16(ref), ref), d)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("merge", [False, True])
@pytest.mark.parametrize("Nk", [300, 257])
def test_attention_planted_defects_fail(Nk, merge):
    B, H, Nq = 2, 2, 40
    _, (q, k, v) = P.att_build(B, H, Nq, Nk, pad=8, merge=merge)
    ref, slack = P.att_reference(q, k, v, B, H, Nq, Nk)
    nb = -(-Nk // 128)
    parts = [(i * nb // 2, (i + 1) * nb // 2) for i in range(2)]        # attn_item's block-aligned KV parts
    if merge:      # the two markers of every code: the first and the last block, so different parts for any split
        for b in range(B):
            for h in range(H):
                for c in range(1, 64):
                    blocks = {j // 128 for j in P.att_markers(b, h, c, Nk, merge=True)}
                    assert blocks == {0, nb - 1}, (b, h, c, blocks)

    def rr(out):
        return P.ratio(r16(out), ref, 1.0, slack)
    model = rr(P.att_blockwise(q, k, v, B, H, Nq, Nk, parts))
    assert model <= EXACT_MAX, model
    d = {name: rr(P.att_blockwise(q, k, v, B, H, Nq, Nk, parts, defect=name)) for name in ("pad", "alpha", "combine")}
    marks = torch.nonzero((k.double().reshape(B * Nk, H, 64)[..., 1:] > 0).any(-1).any(-1)).flatten() % Nk
    drop, dbl = [], []
    for j in sorted(set(marks.tolist())):
        drop.append(rr(P.att_blockwise(q, k, v, B, H, Nq, Nk, parts, drop=j)))
        dbl.append(rr(P.att_blockwise(q, k, v, B, H, Nq, Nk, parts, double=j)))
    d.update(drop=min(drop), double=min(dbl))
    # the neighbouring batch's keys in place of this one's
    kx = k.reshape(B, Nk, -1).flip(0).reshape(B * Nk, -1)
    d["batch"] = rr(P.att_reference(q, kx, v, B, H, Nq, Nk)[0])
    report(f"attention Nk{Nk} merge{merge}", rr(ref), d)


@pytest.mark.parametrize("Nk,n_ip,ip_scale", [(81, 4, 0.6), (128, 16, 1.0), (33, 32, 0.6), (81, 1, 1.0)])
def test_attention_two_segment_planted_defects_fail(Nk, n_ip, ip_scale):
    B, H, Nq = 2, 2, 40
    _, (q, k, v) = P.att_build(B, H, Nq, Nk, n_ip=n_ip)
    ref, slack = P.att_reference(q, k, v, B, H, Nq, Nk, n_ip, ip_scale)

    def rr(out):
        return P.ratio(r16(out), ref, 1.0, slack)
    nt = Nk - n_ip
    zk = torch.zeros(B * 1, k.shape[1], dtype=k.dtype)
    # a zero-filled padding key let into the image-prompt segment
    kp = torch.cat([k.reshape(B, Nk, -1), zk.reshape(B, 1, -1)], 1).reshape(B * (Nk + 1), -1)
    vp = torch.cat([v.reshape(B, Nk, -1), zk.reshape(B, 1, -1)], 1).reshape(B * (Nk + 1), -1)
    d = {"pad": rr(P.att_reference(q, kp, vp, B, H, Nq, Nk + 1, n_ip + 1, ip_scale)[0])}
    if n_ip > 1:     # the text | image-prompt boundary one key late
        d["seam"] = rr(P.att_reference(q, k, v, B, H, Nq, Nk, n_ip - 1, ip_scale)[0])
    report(f"attention two-segment Nk{Nk} ip{n_ip} s{ip_scale}", rr(ref), d)
    assert nt >= 1


# ---------------------------------------------------------------------------------------------------------------------
# guidance rescale
# ---------------------------------------------------------------------------------------------------------------------
def _check_ratio(out, ref, rtol=2e-3, atol=2e-3):
    """test_kernels_gpu.check's bar as a ratio (census.check_ratio)."""
    return float(((out - ref).abs() / (atol + rtol * ref.abs() + ref.abs() * 2.0 ** -11)).max())


@pytest.mark.parametrize("guidance", [5.0, 7.5])
@pytest.mark.parametrize("n,h,w", [(3, 64, 48), (3, 128, 128), (1, 104, 152)])
def test_rescale_planted_defects_fail(n, h, w, guidance):
    noise = P.rescale_build(n, h, w)
    flat = noise.reshape(2 * n, -1)
    assert bool((flat[:, 0] != 0).all() and (flat[:, -1] != 0).all()), "every image marks its first and last element"
    ref = P.rescale_eps(noise, guidance, 0.7)
    dims = (1, 2, 3)

    def std_skip(u, c, g, which, mult, b, j):
        c2, g2 = c.clone(), g.clone()
        for t, on in ((c2, which in ("text", "both")), (g2, which in ("cfg", "both"))):
            if on:
                t.reshape(t.shape[0], -1)[b, j] *= mult
        return c2.std(dim=dims, keepdim=True), g2.std(dim=dims, keepdim=True)
    d = {}
    u0, c0 = noise.double().chunk(2)
    g0 = u0 + guidance * (c0 - u0)
    # an element skipped in (mult 0) or counted twice in (mult sqrt 2) the text sums, the guided sums, or both: the
    # kernels accumulate all four sums in one loop
    for which in ("text", "cfg", "both"):
        src = {"text": c0, "cfg": g0, "both": c0.abs() + g0.abs()}[which]
        for b in range(n):
            marks = torch.nonzero(src.reshape(n, -1)[b]).flatten().tolist()
            for name, mult in (("drop", 0.0), ("double", 2.0 ** 0.5)):
                r = min(_check_ratio(r16(P.rescale_eps(
                    noise, guidance, 0.7, lambda u, c, g: std_skip(u, c, g, which, mult, b, j))), ref) for j in marks)
                d[f"{name}-{which}"] = min(d.get(f"{name}-{which}", float("inf")), r)
    if n > 1:
        d["image"] = _check_ratio(r16(P.rescale_eps(noise, guidance, 0.7, lambda u, c, g: (
            c.std(dim=dims, keepdim=True).roll(1, 0), g.std(dim=dims, keepdim=True).roll(1, 0)))), ref)
    report(f"rescale n{n} {h}x{w} s{guidance}", _check_ratio(r16(ref), ref), d)
