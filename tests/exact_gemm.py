"""Exact-arithmetic operands for the tensor-core GEMM (gemm_f16_kernel, gemm_pp_f16_kernel) and the implicit-GEMM 3x3
convolution.

Gaussian operands against a relative bar let a single lost product, a stale K element, a slightly wrong LayerNorm
`1/K` or one channel read from the wrong tap pass.  Here every operand is a small integer in fp16, so every product is
an integer, every fp32 partial sum an integer far below 2^24, and every epilogue term (bias, row bias, residual, the
power-of-two alpha) exactly representable: the accumulator does not depend on k-block order, ring stage or
tensor-core rounding, and the stored fp16 value must equal fp16(fp64 reference) bit for bit.  With |y| <= 2048 every
+-1 change of an accumulator is a different fp16 value, so a dropped, doubled, stale or misaddressed product fails at
the element it touched.

Where the epilogue evaluates a function that is not exact (the LayerNorm fold's rsqrtf, GELU's erf_as, the __expf of
SiLU and QuickGELU) the bar is 1 fp16 ulp of the fp64 reference of the exact pre-activation (planted.ratio), with
magnitudes chosen so that a +-1 error of any accumulator costs at least 4 bars.  GEGLU is held bit for bit too: its
gate pre-activations are kept at |g| >= 8, where erf_as rounds to +-1 in fp32 and value * gelu(gate) is value * gate
or 0, both exact.

Builders are deterministic and device-agnostic (integer hashes, built on `device`).  Each reference takes a `defect`
that models a broken kernel; test_exact_gemm_cpu.py shows each defect fails its case, test_exact_gemm_gpu.py runs the
kernels.
"""
import torch

from planted import ratio

BK = 64
NUM_SMS = 132            # H100 SXM; the GPU tests pass the device's own count
SENTINEL = 1234.0        # fp16-exact value of the memory around output windows

# gemm_f16_kernel instantiations (gemm.cu dispatch): tile width -> stages.  GEGLU widths count the B tile's rows.
PLAIN_STAGES = {64: 8, 128: 6, 160: 5, 192: 4, 256: 4}
GEGLU_STAGES = {128: 6, 192: 5, 256: 4}


# ---------------------------------------------------------------------------------------------------------------------
# integer operands
# ---------------------------------------------------------------------------------------------------------------------
def _mix(h):
    h = h & 0x7FFFFFFF
    h = ((h ^ (h >> 15)) * 0x2C1B3C6D) & 0x7FFFFFFF
    h = ((h ^ (h >> 12)) * 0x297A2D39) & 0x7FFFFFFF
    return h ^ (h >> 15)


def _hash(rows, cols, seed, device):
    r = torch.arange(rows, device=device, dtype=torch.int64)[:, None]
    c = torch.arange(cols, device=device, dtype=torch.int64)[None, :]
    return _mix(_mix(r * 40503 + seed * 1000003 + 17) + c * 69069)


def seam_cols(K):
    """The first and the last column of every 64-wide k-block, and the last column (the K tail)."""
    k = torch.arange(K)
    return k[(k % BK == 0) | (k % BK == BK - 1) | (k == K - 1)]


def ints(rows, cols, lo, hi, seed, device="cpu", nonzero=None):
    """fp64 [rows, cols] of integers in [lo, hi]; at the columns `nonzero` (a bool mask or index tensor, or True for
    all) a zero becomes +-1."""
    h = _hash(rows, cols, seed, device)
    v = (lo + h % (hi - lo + 1)).double()
    if nonzero is not None:
        mask = torch.zeros(cols, dtype=torch.bool, device=device)
        mask[nonzero if nonzero is not True else slice(None)] = True
        pm = 1.0 - 2.0 * ((h >> 7) & 1).double()
        v = torch.where(mask[None, :] & (v == 0), pm, v)
    return v


def dense(rows, cols, seed, amp=1, device="cpu"):
    """fp16 integers in [-amp, amp], nonzero on every k-block seam (seam_cols)."""
    return ints(rows, cols, -amp, amp, seed, device, nonzero=seam_cols(cols).to(device)).half()


def sparse_rows(rows, K, L, seed, device="cpu", signs="pm", n_neg=2):
    """fp16 [rows, K] with L unit entries per row (coinciding positions add up: the row's L1 norm stays <= L).  Row n
    takes 8 k-block seams, rotating through seam_cols(K) with n, and L - 8 hashed positions, so every seam of every
    k-block is a nonzero of some row in every 64-row stretch.  signs: "pm" hashed +-1; "pos" +1 but the first n_neg
    entries -1 (row sums >= -n_neg with a nonnegative A); "pairs" +1 / -1 alternately (zero row sum, L even)."""
    seams = seam_cols(K).to(device)
    ns = len(seams)
    n = torch.arange(rows, device=device)[:, None]
    j = torch.arange(L, device=device)[None, :]
    h = _hash(rows, L, seed, device)
    pos = torch.where(j < 8, seams[(n * 8 + j * 5 + seed) % ns], h % K)
    if signs == "pm":
        val = 1.0 - 2.0 * ((h >> 9) & 1).double()
    elif signs == "pos":
        val = torch.where(j < n_neg, -1.0, 1.0).double().expand(rows, L)
    else:
        assert L % 2 == 0
        val = torch.where(j % 2 == 0, 1.0, -1.0).double().expand(rows, L)
    w = torch.zeros(rows, K, dtype=torch.float64, device=device)
    w.scatter_add_(1, pos, val)
    return w.half()


def ln_rows(rows, K, seed, device="cpu"):
    """fp16 raw LayerNorm input rows: off[m] + s[m] u[m, k], off in {-1, 0, 1}, s in {1, 2}, u in {-1, 0, 1} nonzero
    on the seams, so rows differ in mean and in std (a statistic read from the neighbouring row shows)."""
    m = torch.arange(rows, device=device, dtype=torch.int64)[:, None]
    off = (_mix(m * 7 + seed) % 3 - 1).double()
    s = (1 + _mix(m * 11 + seed + 5) % 2).double()
    return (off + s * ints(rows, K, -1, 1, seed + 1, device, nonzero=seam_cols(K).to(device))).half()


def slab_stats(x):
    """fp32 [ceil(K / 64), M, 2] per-64-column (sum, sum of squares) of the rows of x: exact for integer rows."""
    M, K = x.shape
    ns = -(-K // BK)
    xd = torch.zeros(M, ns * BK, dtype=torch.float64, device=x.device)
    xd[:, :K] = x.double()
    xd = xd.view(M, ns, BK)
    st = torch.stack([xd.sum(-1), (xd * xd).sum(-1)], -1).transpose(0, 1).contiguous()
    assert float(st.abs().max()) < 2 ** 24
    return st.float()


def vec(n, lo, hi, seed, device="cpu"):
    return ints(1, n, lo, hi, seed, device)[0].half()


# ---------------------------------------------------------------------------------------------------------------------
# GEMM: one case = operands + epilogue
# ---------------------------------------------------------------------------------------------------------------------
ACTS = {None: lambda t: t,
        "silu": torch.nn.functional.silu,
        "gelu": torch.nn.functional.gelu,
        "quick_gelu": lambda t: t * torch.sigmoid(1.702 * t)}


def gemm_case(M, N, K, *, seed=0, bias=False, rowbias=False, rows_per_group=0, residual=False, act=None, alpha=1.0,
              relu=False, geglu=False, ln=False, stats=False, device="cpu"):
    """Operands of one exact GEMM case (a dict; N counts the weight rows, 2 x the outputs for GEGLU).
    Plain: A and W dense in [-1, 1].  Activations: A in {0, 1}, W rows of 11 ones and 5 minus ones (the minus ones
    and 3 ones on k-block seams, where A is 1), bias and row bias in {0, 1}: pre-activations in [-2, 8], where SiLU / GELU / QuickGELU move by >= 4 ulps per unit and GELU's
    erf_as is within a fraction of an ulp.  GEGLU: value rows 12 +-1, gate rows 24 +-1, gate bias +-(32..40) (ln:
    +-(56..64)).  LayerNorm fold: raw rows ln_rows, W rows of 16 +1 / -1 pairs (zero row sum: the centring is exact),
    statistics slab_stats."""
    n_out = N // 2 if geglu else N
    c = {"M": M, "N": N, "K": K, "geglu": geglu, "act": act, "alpha": alpha, "relu": relu, "ln": ln,
         "rows_per_group": rows_per_group if rowbias else 0, "eps": 1e-5}
    if act is not None:
        c["a"] = ints(M, K, 0, 1, seed, device, nonzero=seam_cols(K).to(device)).abs().half()
        c["w"] = sparse_rows(N, K, 16, seed + 1, device, signs="pos", n_neg=5)
        blo, bhi = 0, 1
    elif ln:
        c["a"] = ln_rows(M, K, seed, device)
        c["w"] = sparse_rows(N, K, 16, seed + 1, device, signs="pairs") if not geglu else None
        blo, bhi = -2, 2
    else:
        c["a"] = dense(M, K, seed, 1, device)
        c["w"] = dense(N, K, seed + 1, 1, device) if not geglu else None
        blo, bhi = -3, 3
    if geglu:
        kind = "pairs" if ln else "pm"
        c["w"] = torch.cat([sparse_rows(n_out, K, 12, seed + 2, device, kind),
                            sparse_rows(n_out, K, 24, seed + 3, device, kind)])
        g0 = 56 if ln else 32
        gate = vec(n_out, 0, 8, seed + 4, device).double() + g0
        sign = 1.0 - 2.0 * (torch.arange(n_out, device=device) * 5 // 3 % 2).double()
        c["bias"] = torch.cat([vec(n_out, -2, 2, seed + 5, device).double(), sign * gate]).half()
    elif bias:
        c["bias"] = vec(N, blo, bhi, seed + 5, device)
    if rowbias:
        groups = -(-M // rows_per_group)
        c["rowbias"] = ints(groups, n_out, blo, bhi, seed + 6, device).half()
    if residual:
        r = 1 if act is not None else 4    # activation cases: a small residual keeps the output's ulp fine
        c["residual"] = ints(M, n_out, -r, r, seed + 7, device).half()
    if ln:
        c["ln_stats"] = slab_stats(c["a"])
    c["stats"] = stats
    return c


def kblock_acc(a, w, defect=None, stages=None, kb=None):
    """fp64 A W^T summed k-block by k-block; defects: "drop" / "double" k-block kb, "stale" k-block kb read as
    kb - stages (a ring stage not yet refilled), "other_tile" k-block kb taken from the A rows of the next 128-row
    tile (the other warpgroup's tile), "k_tail" the first column past K let in as the A column of a poisoned window."""
    ad, wd = a.double(), w.double()
    K = a.shape[1]
    nkb = -(-K // BK)
    if defect is None:
        return ad @ wd.t()
    kb = nkb - 1 if kb is None else kb
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64, device=a.device)
    for j in range(nkb):
        s = slice(j * BK, min(K, (j + 1) * BK))
        part = ad[:, s] @ wd[:, s].t()
        if j == kb and defect == "stale":
            assert j >= stages
            part = ad[:, (j - stages) * BK:(j - stages + 1) * BK] @ wd[:, (j - stages) * BK:(j - stages + 1) * BK].t()
        elif j == kb and defect == "other_tile":
            part = ad.roll(-128, 0)[:, s] @ wd[:, s].t()
        elif j == kb and defect == "drop":
            part = part * 0
        elif j == kb and defect == "double":
            part = part * 2
        acc = acc + part
    if defect == "k_tail":
        acc = acc + float("nan") * wd[:, :1].t()
    return acc


def gemm_ref(c, defect=None, stages=None, kb=None):
    """(fp64 output [M, n_out], fp64 exact pre-activation accumulators of the epilogue).  Defects: those of kblock_acc,
    and "geglu_swap" (value and gate halves swapped), "gate_group" (the gate of column n taken from column n + 8),
    "rowbias_group" (row-bias group + 1), "residual_row" (residual of the next row), "alpha_bias" (alpha applied to
    the bias), "ln_inv_c" (1 / (K + 8)), "ln_row" (rstd of the next row)."""
    M, N, K = c["M"], c["N"], c["K"]
    acc = kblock_acc(c["a"], c["w"], defect, stages, kb)
    scale = torch.full((M, 1), float(c["alpha"]), dtype=torch.float64, device=acc.device)
    if c["ln"]:
        st = c["ln_stats"].double().sum(0)
        inv_c = 1.0 / (K + 8 if defect == "ln_inv_c" else K)
        mean = st[:, 0] * inv_c
        var = (st[:, 1] * inv_c - mean * mean).clamp_min(0)
        rstd = 1.0 / torch.sqrt(var + c["eps"])
        if defect == "ln_row":
            rstd = rstd.roll(-1, 0)
        scale = scale * rstd[:, None]
    b = c["bias"].double() if "bias" in c else torch.zeros(N, dtype=torch.float64, device=acc.device)
    x = scale * acc + (scale * b if defect == "alpha_bias" else b)
    mag = (scale * acc).abs() + b.abs()     # the terms' magnitude: the fp32 slack of the 1-ulp cases
    pre = acc
    if c["geglu"]:
        n = N // 2
        v, g = x[:, :n], x[:, n:]
        if defect == "geglu_swap":
            v, g = g, v
        if defect == "gate_group":
            g = g.roll(-8, 1)
        x = v * torch.nn.functional.gelu(g)
        mag = mag[:, :n] * mag[:, n:]
    if "rowbias" in c:
        rpg = c["rows_per_group"]
        grp = torch.arange(M, device=acc.device) // rpg + (1 if defect == "rowbias_group" else 0)
        rb = c["rowbias"].double()[grp.clamp_max((M - 1) // rpg)]
        x, mag = x + rb, mag + rb.abs()
    if c["act"] is not None:
        pre = x
        x = ACTS[c["act"]](x)
        mag = mag.maximum(x.abs())
    if "residual" in c:
        r = c["residual"].double()
        x = x + (r.roll(-1, 0) if defect == "residual_row" else r)
        mag = mag + r.abs()
    if c["relu"]:
        x = x.clamp_min(0)
    if defect is None:
        # fp32 evaluation of rsqrtf, the statistics, erf_as and __expf, and the sum of the epilogue's terms: a few
        # fp32 ulps of the largest term, far below any +-1 accumulator error (test_exact_gemm_cpu checks both)
        c["slack"] = 2.0 ** -19 * mag
    return x, pre


def gemm_exact(c):
    """Whether the case is held bit for bit (everything but the LayerNorm fold and the transcendental activations)."""
    return not c["ln"] and c["act"] is None


def gemm_check_bounds(c, ref, pre):
    """The exactness claims of a case: every fp32 partial sum of every output is an integer below 2^24 (sum |a| |w|),
    bitwise cases stay within |y| <= 2048 (every +-1 is another fp16 value), GEGLU gates within |g| >= 8."""
    l1 = c["a"].double().abs() @ c["w"].double().abs().t()
    assert float(l1.max()) < 2 ** 24
    if gemm_exact(c):
        assert float(ref.abs().max()) <= 2048, float(ref.abs().max())
    if c["geglu"]:
        gate = _gate_pre(c)
        assert float(gate.abs().min()) >= 8, float(gate.abs().min())
    if c["act"] is not None:
        assert float(pre.min()) >= -3 and float(pre.max()) <= 64, (float(pre.min()), float(pre.max()))


def _gate_pre(c):
    """fp64 gate pre-activations rstd * acc + gate bias of a GEGLU case."""
    n = c["N"] // 2
    acc = c["a"].double() @ c["w"][n:].double().t()
    scale = float(c["alpha"])
    if c["ln"]:
        st = c["ln_stats"].double().sum(0)
        mean = st[:, 0] / c["K"]
        scale = scale / torch.sqrt((st[:, 1] / c["K"] - mean * mean).clamp_min(0) + c["eps"])[:, None]
    return scale * acc + c["bias"][n:].double()


def check_bits(out, ref):
    """Number of elements whose fp16 output differs from fp16(ref) (NaN counts as different; -0 equals +0)."""
    want = ref.half()
    bad = ~(out == want) | ~torch.isfinite(out)
    return int(bad.sum())


def gemm_bar(out, c, ref):
    """(mismatching elements, None) for bitwise cases, (None, max err / bar) for the others: 1 fp16 ulp of the fp64
    reference plus gemm_ref's fp32 slack (which matters where terms cancel, as a residual against the product)."""
    if gemm_exact(c):
        return check_bits(out, ref), None
    return None, ratio(out, ref, 1.0, c.get("slack"))


def first_mismatch(out, ref, bn_out=None):
    """Where a bitwise case first fails: element, tile and values, for the assertion message."""
    bad = ~(out == ref.half()) | ~torch.isfinite(out)
    if not bool(bad.any()):
        return None
    idx = bad.nonzero()[0].tolist()
    msg = {"element": idx, "got": float(out[tuple(idx)]), "want": float(ref[tuple(idx)]), "count": int(bad.sum())}
    if bn_out and len(idx) == 2:
        msg["tile"] = (idx[0] // 128, idx[1] // bn_out)
    return msg


# ---------------------------------------------------------------------------------------------------------------------
# stats_out: per-row (sum, sum of squares) slots of the stored fp16 values
# ---------------------------------------------------------------------------------------------------------------------
def stats_model(out16, bn_out, defect=None):
    """The slot layout gemm_f16_kernel writes (fp64 [ceil(N / 64), M, 2], NaN where no slab is written): one slot per
    64 columns; a 160-column tile pair covers its 320 columns' five slots, the odd tile's slab 0 carried into slot 4 of
    the pair with its slab 2.  Defects: "slot_missing" (slot 1 never written), "wrong_slot" (slot 1's values written
    into slot 2), "lost_carry" (the odd 160-column tile's slab 0 dropped)."""
    M, N = out16.shape
    x = out16.double()
    ns = -(-N // 64)
    slots = torch.full((ns, M, 2), float("nan"), dtype=torch.float64, device=out16.device)
    for s in range(ns):
        blk = x[:, s * 64:(s + 1) * 64]
        slots[s, :, 0], slots[s, :, 1] = blk.sum(1), (blk * blk).sum(1)
    if bn_out == 160 and defect == "lost_carry":
        for base in range(0, ns, 5):
            if base + 2 < ns:   # the odd tile's slab 0 is columns 160..223: slot 2's second half
                blk = x[:, (base * 64) + 160:(base * 64) + 192]
                slots[base + 2, :, 0] -= blk.sum(1)
                slots[base + 2, :, 1] -= (blk * blk).sum(1)
    if defect == "slot_missing":
        slots[1] = float("nan")
    if defect == "wrong_slot":
        slots[2] = slots[1]
        slots[1] = float("nan")
    return slots


def stats_totals(out16):
    """(fp64 [M, 2] row (sum, sum of squares) of the stored fp16 values, the allowance of an fp32 sum of them).  Integer
    outputs (every case but the LayerNorm fold's) have exact fp32 sums: the allowance is 0, and the builder asserts
    they stay below 2^24."""
    x = out16.double()
    t = torch.stack([x.sum(1), (x * x).sum(1)], -1)
    if bool((x == x.round()).all()):
        assert float((x * x).sum(1).max()) < 2 ** 24, "row sum of squares beyond fp32's exact integers"
        return t, torch.zeros_like(t)
    return t, 2.0 ** -20 * torch.stack([x.abs().sum(1), (x * x).sum(1)], -1)


def stats_bad(slots, out16):
    """Rows whose slot totals differ from the row totals (NaN in any slot counts as different)."""
    tot = slots.double().sum(0)
    want, tol = stats_totals(out16)
    return int((~((tot - want).abs() <= tol)).any(-1).sum())


# ---------------------------------------------------------------------------------------------------------------------
# the kernels' tile choices, restated
# ---------------------------------------------------------------------------------------------------------------------
def pick_bn(m_tiles, N, num_kb, allow160, sms=NUM_SMS):
    """gemm.cu pick_bn."""
    if N <= 64:
        return 64
    if m_tiles * (-(-N // 64)) <= sms:
        return 64
    best, best_bn = 1e30, 256
    for bn, kbc, fc in ((256, 1.99, 15.1), (192, 1.50, 6.7), (160, 1.21, 6.3), (128, 1.0, 5.7)):
        if bn == 160 and not allow160:
            continue
        rounds = -(-(m_tiles * (-(-N // bn))) // sms)
        t = rounds * (kbc * num_kb + fc)
        if t < best - 1e-9:
            best, best_bn = t, bn
    return best_bn


def pick_bw(Ho, Wo):
    """conv_impl's spatial tile: bw x (128 / bw) output pixels, the fewest tiles, the widest on ties."""
    best_bw, best = 128, -1
    bw = 128
    while bw >= 1:
        t = -(-Wo // bw) * -(-Ho // (128 // bw))
        if best < 0 or t < best:
            best, best_bw = t, bw
        bw >>= 1
    return best_bw


def conv_tiles(B, Ho, Wo, Cout, bn):
    bw = pick_bw(Ho, Wo)
    return B * -(-Wo // bw) * -(-Ho // (128 // bw)) * -(-Cout // bn)


# ---------------------------------------------------------------------------------------------------------------------
# GPU case lists (shared with the CPU self-test's coverage claims)
# ---------------------------------------------------------------------------------------------------------------------
def ring_cases():
    """(geglu, tile, stages, num_kb, tiles per CTA, K % 64) for every gemm_f16_kernel instantiation: num_kb at 1,
    STAGES - 1, STAGES, STAGES + 1 and 2 STAGES + 1 (co-prime), at 0.5, 1.5 and 3 tiles per CTA, the K tail rotating
    through 0, 8 and 56."""
    out = []
    for geglu, table in ((False, PLAIN_STAGES), (True, GEGLU_STAGES)):
        for bn, st in table.items():
            for kb in sorted({1, st - 1, st, st + 1, 2 * st + 1}):
                for i, per_cta in enumerate((0.5, 1.5, 3)):
                    out.append((geglu, bn, st, kb, per_cta, (0, 8, 56)[(kb + i) % 3]))
    return out


def ring_shape(geglu, bn, kb, per_cta, tail, sms=NUM_SMS):
    """(M, N weight rows, K) of a ring case: 3 column tiles, the last ragged by 24 outputs; ceil(tiles / 3) row tiles,
    the last ragged by 37 rows."""
    bn_out = bn // 2 if geglu else bn
    tiles = max(1, int(per_cta * sms))
    n_out = 3 * bn_out - 24
    M = 128 * -(-tiles // 3) - 37
    K = 64 * kb if tail == 0 else 64 * (kb - 1) + tail
    return M, (2 * n_out if geglu else n_out), K


def ring_class(tiles, sms=NUM_SMS):
    """Tiles per CTA: "<1", "1-2" or ">=3"."""
    return "<1" if tiles < sms else ("1-2" if tiles < 3 * sms else ">=3")


# epilogue combinations of the API: (name, kwargs of gemm_case).  Scaled launches (alpha / relu) cannot force a tile:
# their shapes come from scaled_shape.
PLAIN_EPILOGUES = [
    ("none", {}),
    ("bias", dict(bias=True)),
    ("bias_rowbias", dict(bias=True, rowbias=True)),
    ("bias_residual", dict(bias=True, residual=True)),
    ("rowbias_residual", dict(rowbias=True, residual=True)),
    ("bias_rowbias_residual", dict(bias=True, rowbias=True, residual=True)),
    ("silu_bias", dict(act="silu", bias=True)),
    ("gelu_bias_residual", dict(act="gelu", bias=True, residual=True)),
    ("quick_gelu_rowbias", dict(act="quick_gelu", rowbias=True)),
    ("silu_rowbias_residual", dict(act="silu", rowbias=True, residual=True, bias=True)),
    ("gelu", dict(act="gelu")),
    ("ln_bias", dict(ln=True, bias=True)),
    ("ln_rowbias_residual", dict(ln=True, bias=True, rowbias=True, residual=True)),
    ("stats_bias_residual", dict(stats=True, bias=True, residual=True)),
    ("stats_rowbias", dict(stats=True, rowbias=True)),
    ("ln_stats", dict(ln=True, stats=True, bias=True)),
]
SCALED_EPILOGUES = [
    ("alpha_bias_residual", dict(alpha=0.25, bias=True, residual=True)),
    ("alpha_gelu_bias", dict(alpha=0.125, act="gelu", bias=True)),
    ("alpha_silu_residual", dict(alpha=0.5, act="silu", residual=True)),
    ("alpha_quick_gelu_bias", dict(alpha=0.25, act="quick_gelu", bias=True)),
    ("relu_alpha_bias_residual", dict(alpha=0.5, relu=True, bias=True, residual=True)),
    ("relu", dict(relu=True)),
]
GEGLU_EPILOGUES = [
    ("bias", {}),
    ("bias_rowbias_residual", dict(rowbias=True, residual=True)),
    ("ln", dict(ln=True)),
    ("stats", dict(stats=True)),
    ("ln_stats_residual", dict(ln=True, stats=True, residual=True)),
]


def epilogue_shape(geglu, bn, i):
    """(M, N weight rows, K, rows_per_group) of the epilogue case i on a forced tile: 2-3 column tiles (N % 320 == 0
    for the 160-column tile's statistics), 981 rows (rows_per_group 200: group seams inside tiles, not dividing M),
    K tails 8 / 56 / 0."""
    bn_out = bn // 2 if geglu else bn
    n_out = 640 if bn_out == 160 else 2 * bn_out + (64 if bn_out % 64 == 0 else 32)
    K = (320 + 8, 384 - 8, 256)[i % 3]
    return 981, (2 * n_out if geglu else n_out), K, 200


def scaled_shape(bn):
    """(M, N, K) at which pick_bn (no statistics: 160 allowed) chooses tile `bn` for an H100's 132 SMs, with more
    tiles than SMs.  The 256-column tile is never its choice for a plain launch (two 128-column tiles cost less), so
    scaled launches reach 64 / 128 / 160 / 192."""
    if bn == 64:
        return 128 * 200 - 19, 56, 64 * 5 - 8
    for kb in (5, 10, 20):
        for m_tiles in range(1, 40):
            for N in range(64, 1600, 64):
                if pick_bn(m_tiles, N, kb, True) == bn and m_tiles * -(-N // bn) > 132:
                    return 128 * m_tiles - 19, N + (8 if N + 8 <= bn * -(-N // bn) else 0), 64 * kb - 8
    raise AssertionError(bn)


# tile_n = 0 at the SDXL UNet / refiner / VAE shapes: (name, M, N, K, kwargs)
SDXL_AUTO = [
    ("unet_proj_out_64x64", 2 * 4096, 640, 640, dict(bias=True, residual=True)),
    ("unet_ff_out_32x32", 2 * 1024, 1280, 5120, dict(bias=True, residual=True)),
    ("unet_geglu_32x32", 2 * 1024, 10240, 1280, dict(ln=True, geglu=True)),
    ("unet_qkv_64x64", 2 * 4096, 1920, 640, dict(ln=True)),
    ("refiner_geglu_32x32", 2 * 1024, 12288, 1536, dict(ln=True, geglu=True)),
    ("refiner_attn_out_16x16", 2 * 256, 1536, 1536, dict(bias=True, residual=True)),
    ("vae_attn_qkv_128x128", 16384, 1536, 512, dict(bias=True)),
    ("vae_time_emb_rowbias", 2 * 4096, 320, 1280, dict(bias=True, rowbias=True)),
]


# ---------------------------------------------------------------------------------------------------------------------
# 3x3 convolution
# ---------------------------------------------------------------------------------------------------------------------
def conv_input(B, H, W, C, seed, device="cpu"):
    """fp16 NHWC integers in {-2, -1, 1, 2}: every pixel nonzero, so a halo read as a wrapped row shows."""
    v = ints(B * H * W, C, -2, 1, seed, device)
    return torch.where(v >= 0, v + 1, v).half().view(B, H, W, C)


def conv_weight(Cout, K, seed, device="cpu"):
    return dense(Cout, K, seed, 1, device)


def selector_weight(Cout, Cin, sc_channels=(), seed=0, device="cpu"):
    """[Cout, 9 Cin + sum(sc_channels)]: output channel co is 3+ picks of +-1 / +-2 at single (tap, channel) columns.
    The picks walk every (tap, channel) pair with the channel at either end of a 64-channel block (taps 0-8 of x, and
    the shortcut sources as taps 9, 10) first, then hashed columns."""
    K = 9 * Cin + sum(sc_channels)
    targets = []
    for t in range(9):
        targets += [t * Cin + c for c in range(Cin) if c % BK in (0, BK - 1)]
    base = 9 * Cin
    for C in sc_channels:
        targets += [base + c for c in range(C) if c % BK in (0, BK - 1)]
        base += C
    P = max(3, -(-len(targets) // Cout) + 1)
    q = torch.arange(Cout * P)
    t = torch.tensor(targets)
    h = _hash(1, Cout * P, seed, "cpu")[0]
    col = torch.where(q < len(targets), t[q.clamp_max(len(targets) - 1)], h % K)
    val = (1.0 + (h >> 5) % 2).double() * (1.0 - 2.0 * ((h >> 9) & 1).double())
    w = torch.zeros(Cout, K, dtype=torch.float64)
    w.index_put_((q % Cout, col), val, accumulate=True)
    return w.half().to(device), set(targets)


def _pix(x, iy, ix, wrap=False):
    """x [B, H, W, C] at integer row / column index grids (zero outside; wrap: the flat row-major pixel index, so a
    column past the edge reads the neighbouring row)."""
    B, H, W, C = x.shape
    if wrap:
        flat = x.reshape(B, H * W, C)
        p = iy[:, None] * W + ix[None, :]
        ok = (p >= 0) & (p < H * W) & (iy[:, None] >= 0) & (iy[:, None] < H)
        return torch.where(ok[None, :, :, None], flat[:, p.clamp(0, H * W - 1)], 0.0)
    ok = (iy[:, None] >= 0) & (iy[:, None] < H) & (ix[None, :] >= 0) & (ix[None, :] < W)
    return torch.where(ok[None, :, :, None], x[:, iy.clamp(0, H - 1)][:, :, ix.clamp(0, W - 1)], 0.0)


def conv_ref(x, w, *, stride=1, pad="all", bias=None, rowbias=None, residual=None, alpha=1.0, relu=False,
             shortcut=(), defect=None, tap=4):
    """fp64 NHWC [B, Ho, Wo, Cout] of the 3x3 convolution (pad 1 on every side, or pad="br": bottom / right only, the
    VAE's Downsample2D) + the 1x1 shortcut over `shortcut` sources, then alpha, bias, row bias [B, Cout], residual,
    ReLU.  Defects: "tap_x+" / "tap_x-" / "tap_y+" / "tap_y-" (tap `tap` shifted by one pixel), "wrap" (halo columns
    read from the neighbouring row), "parity" (the dx = 0 and dx = 2 taps of a stride-2 conv on the other column
    parity), "pad_side" (the other padding), "sc_swap" (shortcut sources swapped), "sc_drop" (the last source
    dropped), "rowbias_group" (the next image's row bias), "residual_row" (the next pixel's residual),
    "alpha_bias" (alpha applied to the bias)."""
    B, H, W, Cin = x.shape
    Ho, Wo = H // stride, W // stride
    xd = x.double()
    wd = w.double()
    p = pad
    if defect == "pad_side":
        p = "br" if pad == "all" else "all"
    acc = torch.zeros(B, Ho, Wo, w.shape[0], dtype=torch.float64, device=x.device)
    oy = torch.arange(Ho, device=x.device)
    ox = torch.arange(Wo, device=x.device)
    for t in range(9):
        dy, dx = t // 3, t % 3
        iy = stride * oy + dy - (1 if p == "all" else 0)
        ix = stride * ox + dx - (1 if p == "all" else 0)
        if t == tap and defect in ("tap_x+", "tap_x-", "tap_y+", "tap_y-"):
            d = 1 if defect[-1] == "+" else -1
            if defect[4] == "x":
                ix = ix + d
            else:
                iy = iy + d
        if defect == "parity" and dx != 1:
            ix = ix + 1
        xs = _pix(xd, iy, ix, wrap=defect == "wrap")
        acc = acc + xs @ wd[:, t * Cin:(t + 1) * Cin].t()
    srcs = list(shortcut)
    offs, o = [], 9 * Cin
    for s in srcs:
        offs.append(o)
        o += s.shape[-1]
    if defect == "sc_swap":
        srcs = srcs[::-1]
    for i, s in enumerate(srcs):
        if defect == "sc_drop" and i == len(srcs) - 1:
            continue
        acc = acc + s.double() @ wd[:, offs[i]:offs[i] + s.shape[-1]].t()
    b = torch.zeros(w.shape[0], dtype=torch.float64, device=x.device) if bias is None else bias.double()
    y = alpha * (acc + b) if defect == "alpha_bias" else alpha * acc + b
    if rowbias is not None:
        rb = rowbias.double()
        if defect == "rowbias_group":
            rb = rb.roll(-1, 0)
        y = y + rb[:B, None, None, :]
    if residual is not None:
        r = residual.double()
        if defect == "residual_row":
            r = r.reshape(B, Ho * Wo, -1).roll(-1, 1).reshape(r.shape)
        y = y + r
    if relu:
        y = y.clamp_min(0)
    return y


def conv_check_bounds(x, w, ref, shortcut=()):
    amax = max([float(x.double().abs().max())] + [float(s.double().abs().max()) for s in shortcut])
    assert float(w.double().abs().sum(1).max()) * amax < 2 ** 24
    assert float(ref.abs().max()) <= 2048, float(ref.abs().max())


# (name, B, H, W, Cin, Cout): SDXL's latent levels at 1024^2 and at the 1216 x 832 bucket, B >= 3 so batch seams fall
# inside the spatial tiling, odd H and W; the spatial tile each gets is pick_bw's
CONV_LEVELS = [
    ("1216x832_l0", 3, 152, 104, 320, 320),
    ("1216x832_l1", 3, 76, 52, 640, 640),
    ("1216x832_l2", 3, 38, 26, 1280, 1280),
    ("1024_l0", 2, 128, 128, 320, 320),
    ("1024_l1", 3, 64, 64, 640, 640),
    ("1024_l2", 3, 32, 32, 1280, 1280),
    ("odd", 3, 37, 23, 128, 192),
]

# one stride-1 shape per spatial tile width bw = 128 ... 1 (Ho, Wo): pick_bw(Ho, Wo) == bw, ragged on both axes
BW_SHAPES = {128: (1, 200), 64: (3, 33), 32: (3, 129), 16: (6, 65), 8: (11, 33), 4: (21, 17), 2: (41, 9), 1: (200, 1)}
SCALED_TILES = (64, 128, 160, 192)

FORCED_TILES = (64, 128, 160, 192, 256)


def conv_tile_cases(sms=NUM_SMS):
    """(tile, B, H, W, Cin, Cout) of ih_conv2d_f16 with every forced tile width at < 1, 1-2 and >= 3 tiles per CTA."""
    out = []
    for bn in FORCED_TILES:
        for target in (0.6, 1.5, 3.2):
            cout = 320 if bn != 192 else 384
            per_img = -(-cout // bn)
            # W = 64: bw 64, two output rows per tile
            rows = max(1, int(target * sms / per_img / 3))
            out.append((bn, 3, 2 * rows - 1, 64, 64, cout))
    return out
