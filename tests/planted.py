"""Planted-marker inputs for the kernels that reduce many elements into one statistic (GroupNorm, LayerNorm, the
attention softmax and its KV-split merge, the masked row softmax, the guidance-rescale std of the step kernels).

Gaussian inputs average a bookkeeping error away: one element dropped from a GroupNorm group of 40960 moves the
output by a tenth of the bar.  Here the background is constant (0, or a constant offset) and a few small-integer
markers sit on the kernels' partition seams, so every fp32 partial sum is exact and the exact result is dominated by
the markers.  One marker lost, counted twice, or credited to the wrong image, row, group, head or key block is then
many fp16 ulps against the fp64 reference, while the kernel itself must land within about one ulp of it.

Builders are deterministic and device-agnostic (they build on `device`); each family has its fp64 reference, the bar
its outputs are held to (as a max err / bar ratio: <= 1 passes) and a defect hook that the CPU self-test
(test_planted_cpu.py) uses to show that a broken kernel would fail.  test_planted_gpu.py runs the kernels.
"""
import math

import torch

from fp16_ulps import ulp_err_tol

NUM_SMS = 132          # H100 SXM; the GPU tests pass the device's own count


def ratio(out, ref, ulps=1.0, slack=None):
    """max(err / bar) of close_ulps' bar (fp16_ulps.py), the same comparator as census.ulp_ratio."""
    if out.shape != ref.shape:
        return float("inf")
    if not bool(torch.isfinite(out).all()):
        return float("inf")
    err, tol = ulp_err_tol(out, ref, ulps, slack)
    return float((err / tol).max().item()) if err.numel() else 0.0


def _sign(i):
    """+-1 from an integer tensor, without a regular pattern a mis-indexed sum could cancel."""
    return 1.0 - 2.0 * ((i * 5 + (i >> 2)) % 3 == 0).double()


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm (ih_groupnorm_f16): NHWC [B, HW, C0 | C1], `groups` groups, optional SiLU
# ---------------------------------------------------------------------------------------------------------------------
GN_PER_GROUP = 32      # markers per (image, group) and launch: one lost ±1 marker moves the group's rstd by >= 1/160
GN_FULL_COVER = 1 << 15  # up to this many rows per image every row is a marker row in some launch; beyond, the seams


# (B, HW, C0, C1, groups, silu, scale) of test_planted_gpu.py: the UNet's levels at 512^2, 1024^2 and 1216x832, the
# up-block concats, B up to 64, 32 / 160 / C/2 groups, the VAE decoder's 1024^2 level (2^-7-scaled stream)
GN_CASES = [
    (2, 4096, 320, 0, 32, True, 1), (2, 1024, 640, 0, 32, False, 1), (2, 256, 1280, 0, 32, True, 1),   # 512^2
    (2, 16384, 320, 0, 32, True, 1), (1, 4096, 640, 0, 32, False, 1), (2, 1024, 1280, 0, 32, True, 1),  # 1024^2
    (2, 15808, 320, 0, 32, False, 1), (2, 3952, 640, 0, 32, True, 1), (2, 988, 1280, 0, 32, True, 1),   # 1216x832
    (2, 1024, 1280, 1280, 32, True, 1), (2, 1024, 1280, 640, 32, True, 1), (2, 4096, 640, 640, 32, True, 1),
    (2, 4096, 640, 320, 32, False, 1), (2, 4096, 320, 320, 32, True, 1),                                 # concats
    (16, 1024, 1280, 0, 32, True, 1), (16, 4096, 320, 0, 32, False, 1), (64, 64, 320, 0, 32, True, 1),
    (2, 1024, 1280, 0, 160, True, 1), (2, 4096, 320, 0, 160, False, 1), (1, 256, 1280, 0, 640, True, 1),
    (3, 1024, 640, 0, 320, False, 1), (2, 1024, 1280, 640, 160, True, 1),
    (1, 1 << 20, 128, 0, 32, True, 2.0 ** -7),                                                           # VAE 1024^2
]


def gn_plan(B, HW, C, num_sms=NUM_SMS):
    """The row-chunk plans of ih_groupnorm_f16 (norm.cu), restated: (R row lanes, rows per block of the two-kernel
    plan, sorted rows per block of the fused plan for every grid size from 1 up to its cap).  The fused grid is capped
    by an occupancy query Python cannot see, so every possible cap is covered."""
    CV = C // 8
    R = max(1, 256 // CV)
    bps = 4 if B >= 8 else 2
    G = min((bps * num_sms + B - 1) // B, 512)
    rpb = max(-(-HW // G), 4 * R)
    fused = sorted({max(-(-HW // g), 4 * R) for g in range(1, G + 1)})
    return R, rpb, fused


def gn_cover_rows(B, HW, C, num_sms=NUM_SMS):
    """Rows each image must have as a marker row in some launch: all of them, or at very large HW the first and last
    row, both sides of every multiple of 4R (the 4-deep unrolled loop against its tail) and of every row-chunk
    boundary of both plans."""
    if HW <= GN_FULL_COVER:
        return torch.arange(HW)
    R, rpb, fused = gn_plan(B, HW, C, num_sms)
    rows = {0, HW - 1}
    for step in [4 * R, rpb] + fused:
        for m in range(step, HW, step):
            rows.update((m - 1, m))
    return torch.tensor(sorted(rows))


def gn_launches(B, HW, C, groups, num_sms=NUM_SMS):
    """Number of launches (different marker sets on one shared workspace) that cover every row to be covered."""
    n = len(gn_cover_rows(B, HW, C, num_sms))
    return max(2, -(-n // (groups * GN_PER_GROUP)))


def gn_seam_channels(C, groups, C0=None):
    """Channels a GroupNorm marker must visit: the first and last channel of every group, both ends of every 8-channel
    vector (the kernels' per-thread load), and C0 - 1 / C0 (the x0 | x1 seam)."""
    c = torch.arange(C)
    cpg = C // groups
    keep = (c % cpg == 0) | (c % cpg == cpg - 1) | (c % 8 == 0) | (c % 8 == 7)
    if C0 is not None and 0 < C0 < C:
        keep |= (c == C0 - 1) | (c == C0)
    return c[keep]


def gn_channel_order(C, groups, C0=None):
    """[groups, cpg] in-group channel offsets, each row a permutation: the group's seam channels (gn_seam_channels)
    first, then the others."""
    cpg = C // groups
    seam = torch.zeros(C, dtype=torch.bool)
    seam[gn_seam_channels(C, groups, C0)] = True
    off = torch.arange(cpg)
    rows = []
    for g in range(groups):
        s = seam[g * cpg:(g + 1) * cpg]
        rows.append(torch.cat([off[s], off[~s]]))
    return torch.stack(rows)


def gn_markers(B, HW, C, groups, launch, n_launch, cover, C0=None):
    """(image, row, channel, value) of launch `launch`.  Image b takes every n_launch-th cover row from offset
    (launch + b) % n_launch, so neighbouring images carry different rows; marker i goes to group (i + 5 launch + 3 b),
    so rows rotate through the groups.  Inside a group the markers walk gn_channel_order: the T = m // groups markers a
    group gets in (launch, image) take positions k T .. k T + T - 1 with k = launch * B + image, so over the launches
    and images every group's seam channels (its ends, both ends of each 8-channel vector, the x0 | x1 seam at C0) are
    visited first and then the rest.  Every group of every image gets at least one marker; values are +-1 and +-2."""
    cpg = C // groups
    order = gn_channel_order(C, groups, C0)
    out = []
    for b in range(B):
        k = (launch + b) % n_launch
        sel = cover[k::n_launch]
        if len(sel) == 0:
            sel = cover[k % len(cover):][:1]
        m = max(len(sel), groups)
        i = torch.arange(m)
        rows = sel[i % len(sel)]
        g = (i + 5 * launch + 3 * b) % groups
        pos = (i // groups + (launch * B + b) * (m // groups)) % cpg
        ch = g * cpg + order[g, pos]
        mag = 1.0 + ((i * 3 + launch + b) % 4 == 0).double()
        out.append((torch.full_like(i, b), rows, ch, _sign(i + 7 * b + launch) * mag))
    return tuple(torch.cat(t) for t in zip(*out))


def gn_params(C, device="cpu"):
    c = torch.arange(C, device=device)
    gamma = (1.0 + ((c * 7) % 9 - 4).double() / 16).half()
    beta = (((c * 5) % 11 - 5).double() / 32).half()
    return gamma, beta


def gn_build(B, HW, C, markers, scale=1.0, device="cpu"):
    """fp16 [B, HW, C]: background 0, the markers times `scale` (a power of two: exact)."""
    b, r, c, v = markers
    x = torch.zeros(B, HW, C, dtype=torch.float16, device=device)
    x[b.to(device), r.to(device), c.to(device)] = (v * scale).half().to(device)
    return x


def gn_sums(x, groups):
    """fp64 (sum, sum of squares) [B, groups]: exact for the marker inputs."""
    B, HW, C = x.shape
    xd = x.double().view(B, HW, groups, C // groups)
    return xd.sum((1, 3)), (xd * xd).sum((1, 3))


def gn_reference(x, gamma, beta, groups, eps, silu, sums=None):
    """(fp64 GroupNorm [+ SiLU] of x, the slack of the kernel's fp32 scale / shift arithmetic).  `sums` replaces the
    statistics (a defect simulation)."""
    B, HW, C = x.shape
    cpg = C // groups
    s, q = gn_sums(x, groups) if sums is None else sums
    n = float(HW * cpg)
    mean = s / n
    var = (q / n - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + eps)
    ga, be = gamma.double(), beta.double()
    sc = rstd.repeat_interleave(cpg, -1)[:, None, :] * ga           # [B, 1, C]
    sh = be - mean.repeat_interleave(cpg, -1)[:, None, :] * sc
    xd = x.double()
    y = xd * sc + sh
    slack = 2.0 ** -20 * ((xd * sc).abs() + sh.abs() + be.abs())
    if silu:
        y = torch.nn.functional.silu(y)
        slack = 1.1 * slack + 2.0 ** -20 * y.abs()
    return y, slack


def gn_check_ratio(out, x, gamma, beta, groups, eps, silu, sums=None):
    ref, slack = gn_reference(x, gamma, beta, groups, eps, silu, sums)
    return ratio(out.reshape(ref.shape), ref, 1.0, slack)


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm (ih_layernorm_f16): rows x C, one 8-column vector per thread, TPR threads per row
# ---------------------------------------------------------------------------------------------------------------------
LN_OFFSET = 4.0


def ln_plan(C):
    """(threads per row, rows per block) of ih_layernorm_f16."""
    TPR = -(-(C // 8) // 32) * 32
    return TPR, max(1, 256 // TPR)


def ln_seam_cols(C):
    """Both ends of every thread's 8-column vector (first / last 64 columns and around every warp seam), both sides of
    every 256-column warp seam, and the last column."""
    cols = {0, 7, C - 1, C - 8}
    for v in range(0, C, 8):
        if v < 64 or v >= C - 64 or v % 256 in (0, 248):
            cols.update((v, v + 7))
    for w in range(256, C, 256):
        cols.update((w - 1, w))
    return torch.tensor(sorted(c for c in cols if 0 <= c < C))


def ln_rows(C, extra):
    """A ragged row count: a few whole blocks plus `extra` rows (so both sides of every block boundary are rows)."""
    _, rpb = ln_plan(C)
    return 3 * rpb + extra


def ln_build(rows, C, seed=0, device="cpu"):
    """fp16 [rows, C]: LN_OFFSET plus 2-5 markers of +-1 / +-2 per row, rotating through the seam columns."""
    seams = ln_seam_cols(C)
    ns = len(seams)
    x = torch.full((rows, C), LN_OFFSET, dtype=torch.float64)
    r = torch.arange(rows)
    for t in range(5):
        use = t < 2 + (r + seed) % 4
        idx = seams[(r * 5 + t * 3 + seed + (t * ns) // 5) % ns]
        mag = 1.0 + ((r + t + seed) % 3 == 0).double()
        x[r[use], idx[use]] += (_sign(r * 5 + t + seed) * mag)[use]
    return x.half().to(device)


def ln_params(C, device="cpu"):
    return gn_params(C, device)


def ln_reference(x, gamma, beta, eps, stats=None):
    """(fp64 LayerNorm, the slack of the kernel's fp32 mean and centring).  `stats` = (mean, var) per row replaces the
    statistics (a defect simulation)."""
    xd = x.double()
    if stats is None:
        mean = xd.mean(-1, keepdim=True)
        var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    else:
        mean, var = stats
    rstd = 1.0 / torch.sqrt(var + eps)
    g, bt = gamma.double(), beta.double()
    y = (xd - mean) * rstd * g + bt
    slack = 2.0 ** -19 * ((xd - mean).abs() + mean.abs()) * rstd * g.abs() + 2.0 ** -22 * bt.abs()
    return y, slack


# ---------------------------------------------------------------------------------------------------------------------
# masked row softmax (ih_softmax_rows_masked_f16): 256 threads x 16 vectors of 8 columns per row
# ---------------------------------------------------------------------------------------------------------------------
SMX_TOP, SMX_BACK, SMX_PAD = 2.0, -28.0, 60000.0


def smx_seam_cols(valid):
    """Both ends of 8-column vectors near the row ends and the thread / vector-loop seams (2048 columns: 256 threads of
    one 8-column vector), and valid - 1."""
    cols = {0, 7, 8, valid - 1}
    for v in range(0, valid, 8):
        if v < 32 or v >= valid - 32 or v % 2048 in (0, 2040):
            cols.update((v, v + 7))
    for s in range(2048, valid, 2048):
        cols.update((s - 1, s))
    return torch.tensor(sorted(c for c in cols if 0 <= c < valid))


def smx_build(rows, cols, valid, ld, device="cpu"):
    """fp16 [rows, ld] and the view [:, :cols].  Valid columns: background SMX_BACK (its softmax weight, e^-30 of a
    maximum's, rounds to fp16 0) and 1-12 tied maxima SMX_TOP at seam columns; columns >= valid hold +SMX_PAD."""
    seams = smx_seam_cols(valid)
    ns = len(seams)
    x = torch.full((rows, ld), SMX_PAD, dtype=torch.float64)
    x[:, :valid] = SMX_BACK
    for r in range(rows):
        k = min(1 + (r * 5) % 12, ns)
        x[r, seams[(r * 7 + torch.arange(k) * max(1, ns // k)) % ns]] = SMX_TOP
    x = x.half().to(device)
    return x, x[:, :cols]


def smx_reference(view, valid):
    """fp64 softmax over the first `valid` columns, 0 beyond."""
    xd = view.double()
    ref = torch.zeros_like(xd)
    ref[:, :valid] = torch.softmax(xd[:, :valid], -1)
    return ref


# ---------------------------------------------------------------------------------------------------------------------
# attention (ih_attention_ws_f16): head dim 64, softmax scale 1/8
# ---------------------------------------------------------------------------------------------------------------------
# q row r of (b, h) has channel 0 = 16 and its code channel c = 16.  Every real key has channel 0 = -16: a baseline of
# -256 / 8 = -32 nats.  A marker key of code c has channel c = 14 (-4 nats) or 14.5 (-3 nats).  A zero-filled padding
# key scores exactly 0 nats and would outweigh every marker by e^3..e^4 if it were let in.  Every score is an exact
# integer before the scale; a baseline key's weight (e^-28 of a marker's) rounds to fp16 0 in the kernel's P.
ATT_Q, ATT_BASE, ATT_MARK, ATT_HI = 16.0, -16.0, 14.0, 14.5


def att_seam_keys(Nk):
    """Key 0, both sides of every 128-key block boundary (the KV-split parts are block-aligned) and Nk - 1."""
    keys = {0, Nk - 1}
    for j in range(128, Nk, 128):
        keys.update((j - 1, j))
    return sorted(keys)


def att_code(b, h, r):
    return 1 + (r + 7 * h + 13 * b) % 63


def att_markers(b, h, c, Nk, merge=False, n_text=None):
    """{key: k value} of code c.  Plain: 1-6 tied markers (-4 nats) at seam keys.  merge: two markers in different
    blocks, the first and the last (so in different KV parts whatever the split), one of them one nat higher, the higher
    one first or last depending on c.  n_text (two-segment path): 1-3 markers in the text keys [0, n_text) and 1-3 in
    the image-prompt keys [n_text, Nk), at n_text - 1, n_text and Nk - 1 among others."""
    seams = att_seam_keys(Nk)
    ns = len(seams)
    if n_text is not None:
        text = sorted({0, n_text - 1} | {(7 * c + 3 * h + b) % n_text})
        out = {text[(c + t) % len(text)]: ATT_MARK for t in range(1 + (c + b) % 3)}
        if Nk > n_text:
            ip = sorted({n_text, Nk - 1} | {n_text + (5 * c + h) % (Nk - n_text)})
            out.update({ip[(c + h + t) % len(ip)]: ATT_MARK for t in range(1 + (c + h) % 3)})
        return out
    if merge:
        # the first and the last key block: in different KV parts for every split (parts are block ranges)
        first = [j for j in seams if j < 128]
        last = [j for j in seams if j >= (Nk - 1) // 128 * 128]
        j1, j2 = first[(c + h + b) % len(first)], last[(c // 2 + h) % len(last)]
        hi = j1 if c % 2 else j2
        return {j1: ATT_MARK, j2: ATT_MARK, hi: ATT_HI}
    k = 1 + (c + h + b) % 6
    return {seams[(c * 7 + h * 3 + b + t * max(1, ns // k)) % ns]: ATT_MARK for t in range(k)}


def att_build(B, H, Nq, Nk, pad=0, merge=False, n_ip=None, device="cpu"):
    """q [B*Nq, H*64 + 2 pad] / k, v [B*Nk, H*64 + 2 pad] buffers (the kernel reads the column views
    [:, pad:pad + H*64]).  The columns outside the views and beyond each row's head hold values that would dominate
    any row that read them: k channel = +16 (+32 nats against q's channel 0), v = 100."""
    W = H * 64 + 2 * pad
    n_text = None if n_ip is None else Nk - n_ip
    q = torch.zeros(B * Nq, W, dtype=torch.float64)
    k = torch.full((B * Nk, W), 16.0, dtype=torch.float64)
    v = torch.full((B * Nk, W), 100.0, dtype=torch.float64)
    r = torch.arange(Nq)
    j = torch.arange(Nk)
    d = torch.arange(64)
    for b in range(B):
        for h in range(H):
            c0 = pad + h * 64
            codes = att_code(b, h, r)
            q[b * Nq + r, c0] = ATT_Q
            q[b * Nq + r, c0 + codes] = ATT_Q
            kb = k[b * Nk:(b + 1) * Nk, c0:c0 + 64]
            kb.zero_()
            kb[:, 0] = ATT_BASE
            for c in set(codes.tolist()):
                for key, val in att_markers(b, h, c, Nk, merge, n_text).items():
                    kb[key, c] = val
            v[b * Nk:(b + 1) * Nk, c0:c0 + 64] = (((j[:, None] * 13 + d * 7 + h * 5 + b * 3) % 31) - 15).double() / 16
    q, k, v = (t.half().to(device) for t in (q, k, v))
    cols = slice(pad, pad + H * 64)
    return (q, k, v), (q[:, cols], k[:, cols], v[:, cols])


def _heads(t, B, N, H):
    return t.double().reshape(B, N, H, 64).transpose(1, 2)


def att_reference(q, k, v, B, H, Nq, Nk, n_ip=0, ip_scale=1.0):
    """(fp64 attention [B*Nq, H*64], the census attention bar's slack 2^-10 (P @ |V|)) of the views q, k, v."""
    qd, kd, vd = _heads(q, B, Nq, H), _heads(k, B, Nk, H), _heads(v, B, Nk, H)
    nt = Nk - n_ip
    p = (qd @ kd[:, :, :nt].transpose(-1, -2) / 8).softmax(-1)
    out, mag = p @ vd[:, :, :nt], p @ vd[:, :, :nt].abs()
    if n_ip:
        pi = (qd @ kd[:, :, nt:].transpose(-1, -2) / 8).softmax(-1)
        out = out + ip_scale * (pi @ vd[:, :, nt:])
        mag = mag + abs(ip_scale) * (pi @ vd[:, :, nt:].abs())
    flat = lambda t: t.transpose(1, 2).reshape(B * Nq, H * 64)   # noqa: E731
    return flat(out), 2.0 ** -10 * flat(mag)


def att_blockwise(q, k, v, B, H, Nq, Nk, parts=None, defect=None, drop=None, double=None):
    """fp64 model of the multi-block kernel: key blocks of 128 (TMA zero-fills the keys past Nk: score 0, v 0), the
    online softmax over the blocks of each KV part, the parts merged with weights e^(m_i - M).  Defects: "pad" lets
    key Nk (the first padding key) in, "alpha" omits the running-max rescale of O and l, "combine" weights part 1
    with part 0's running max; drop / double: a key left out of / counted twice in every row's sums."""
    nb = -(-Nk // 128)
    if parts is None:
        parts = [(0, nb)]
    qd, kd, vd = _heads(q, B, Nq, H), _heads(k, B, Nk, H), _heads(v, B, Nk, H)
    padn = nb * 128 - Nk
    kd = torch.cat([kd, kd.new_zeros(B, H, padn, 64)], 2)
    vd = torch.cat([vd, vd.new_zeros(B, H, padn, 64)], 2)
    s = qd @ kd.transpose(-1, -2) / 8
    valid = torch.arange(nb * 128, device=s.device) < Nk + (1 if defect == "pad" else 0)
    s = s.masked_fill(~valid, -math.inf)
    mult = torch.ones(nb * 128, dtype=torch.float64, device=s.device)
    if drop is not None:
        mult[drop] = 0.0
    if double is not None:
        mult[double] = 2.0
    res = []
    for jb, je in parts:
        m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=torch.float64, device=s.device)
        o = torch.zeros(B, H, Nq, 64, dtype=torch.float64, device=s.device)
        l = torch.zeros_like(m)
        for blk in range(jb, je):
            cols = slice(blk * 128, blk * 128 + 128)
            sb = s[..., cols]
            m_new = torch.maximum(m, sb.amax(-1, keepdim=True))
            alpha = torch.exp(m - m_new).nan_to_num(0.0)
            if defect == "alpha" and blk > jb:
                alpha = torch.ones_like(alpha)
            p = torch.exp(sb - m_new) * mult[cols]
            o = o * alpha + p @ vd[..., cols, :]
            l = l * alpha + p.sum(-1, keepdim=True)
            m = m_new
        res.append((m, l, o))
    M = torch.stack([r[0] for r in res]).amax(0)
    num = torch.zeros_like(res[0][2])
    den = torch.zeros_like(res[0][1])
    for i, (m, l, o) in enumerate(res):
        w = torch.exp((res[0][0] if defect == "combine" and i == 1 else m) - M)
        num, den = num + o * w, den + l * w
    return (num / den).transpose(1, 2).reshape(B * Nq, H * 64)


# ---------------------------------------------------------------------------------------------------------------------
# guidance rescale of the step kernels: per-image std of the text branch and of the guided prediction
# ---------------------------------------------------------------------------------------------------------------------
def rescale_seams(per):
    """First and last element of an image, both sides of the warp and 1024-thread strides, and a few interior
    elements: the seams of the kernels' strided per-image reduction."""
    pos = {0, per - 1, 31, 32, 1023, 1024, 2047, 2048, per - 1024, per - 1025, per // 2, per // 3 + 1}
    return sorted(p for p in pos if 0 <= p < per)


def rescale_build(n, h, w, device="cpu"):
    """noise_pred [2n, 4, h, w] (uncond | text): background 0.  The text branch of every image holds markers of
    +-1.5 and +-1 (alternating) times (1 + image) at its first and last element and at 3-5 of the other seams (rotating
    through them over the images), so that one marker is at least a twelfth of its variance.  The uncond branch equals
    it except at the +-1 markers, which it moves towards 0 by 3/16, 1/4 or 7/32 of (1 + image), by image.
    In the guided prediction u + s (c - u) those markers become the larger ones: every marker has a different share of
    the two variances, so a marker skipped in both std sums still moves their ratio; the guided std is of the text
    branch's order, so the rescale factor carries weight in the result; and the factor differs per image, so a std
    taken over the wrong image shows."""
    per = 4 * h * w
    seams = rescale_seams(per)
    ns = len(seams)
    x = torch.zeros(2 * n, per, dtype=torch.float64)
    inner = seams[1:-1]                                 # every image marks 0 and per - 1; the rest rotate
    for b in range(n):
        k = 3 + b % 3
        sel = torch.tensor(sorted({0, per - 1} | {inner[(t * 3 + b) % len(inner)] for t in range(k)}))
        t = torch.arange(len(sel))
        small = (t + b) % 2 == 1
        text = _sign(t + 3 * b) * (1 + b) * (1.0 + 0.5 * (~small).double())
        x[n + b, sel] = text
        x[b, sel] = text - text.sign() * small.double() * (1 + b) * (0.1875, 0.25, 0.21875)[b % 3]
    return x.half().reshape(2 * n, 4, h, w).to(device)


def rescale_eps(noise_pred, guidance, rescale, std_of=None):
    """fp64 guided prediction with the guidance rescale (oracle.scheduler_ref.rescale_noise_cfg without its fp16
    rounding points).  std_of(u, c, g) -> (std_text, std_cfg) [n, 1, 1, 1] replaces the statistics (a defect)."""
    u, c = noise_pred.double().chunk(2)
    g = u + guidance * (c - u)
    if std_of is None:
        st = c.std(dim=(1, 2, 3), keepdim=True)
        sg = g.std(dim=(1, 2, 3), keepdim=True)
    else:
        st, sg = std_of(u, c, g)
    return rescale * g * (st / sg) + (1 - rescale) * g
