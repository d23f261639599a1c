"""Per-call census of the imagharmony_b200.ops calls a model forward makes (test helper, not a test module).

`Census.install(monkeypatch)` wraps every public function of `ops`.  Each call of an op with a reference is recorded
under a key (op, every tensor argument's shape / stride / dtype, the scalar arguments, and the execution plan the
caller's `plan` hook reports); the op runs, and then a reference computed from the same inputs is compared with what
it produced, against a bar derived from the op's rounding points.  So every layer is checked at its real shape on live
activations, with no error carried over from earlier layers.  A call of an op without a reference raises, so a new op
cannot skip the census; only the host-side helpers in EXEMPT run unchecked.

References are the plain-PyTorch stand-ins of tests/fake_ops.py, evaluated on the inputs' device: GEMM and conv in
fp64 (their bar below has no room for the reference's own accumulation error), everything else in fp32 with TF32 off,
plus the magnitudes the bars need.  Bars (max err / bar <= 1 passes):

* layout ops: bit-exact;
* GEMM / conv, against the unrounded fp64 result: the kernel stores fp16 once, after the whole fp32 epilogue
  (gemm.cu), so half an fp16 ulp, plus
  - the accumulation: the wgmma main loop keeps one fp32 accumulator per output over all of K and adds one k16 MMA
    step to it at a time, ceil(K / 16) roundings of a running sum.  A running sum never exceeds |A| @ |W|^T (the
    products are exact in fp32), and one rounding loses at most one fp32 ulp of it, 2^-23 (a truncating adder; a
    rounding one loses half): ceil(K / 16) * 2^-23 * (|A| @ |W|^T), times alpha and rstd where they scale it;
  - the epilogue in fp32 (fma with the bias, activation, residual add): EPI = 2^-21 of the values it forms, a few
    fp32 roundings and the fp32 erf / exp approximations;
  - both carried through the steepest slope of the activation (1.13 for GELU; SiLU and quick-GELU peak at 1.10);
* the folded-LayerNorm consumer, against both the slot statistics the kernel reads and the true fp64 statistics of
  its raw rows: plus the error of var = E[x^2] - mean^2 from fp32 sums of K terms (the producer's slots and their
  total; each sum off by at most K 2^-24 of its magnitude, the fp16 squares exact in fp32), 3 K 2^-24 E[x^2] /
  (var + eps) relative on var, half of it on rstd, plus 2^-22 for rsqrtf;
* `stats_out` slots: their totals against the row sums of the stored fp16 output in fp64, within N 2^-24 sum|x|
  (resp. sum x^2): any fp32 summation order of N terms;
* attention: P is packed to fp16 before the PV MMA (half an fp16 ulp of every p) and exp / the score sums in fp32 stay
  below another half: 1 ulp + 2^-10 * (P @ |V|), the IP part weighted by |ip_scale|;
* norms, linear_small, sinusoid, masked softmax: the bars of their existing kernel tests, against unrounded fp32.
"""
import inspect

import torch
import torch.nn.functional as F

import fake_ops
from fp16_ulps import ulp_err_tol

EXEMPT = {"prefetch_next", "fold_layernorm", "pack_conv3x3_weight", "workspace_generation", "launch_count"}
ACC_STEP = 2.0 ** -23     # one rounding of the fp32 accumulator per k16 MMA step, relative to |A| @ |W|^T
EPI = 2.0 ** -21          # the fp32 epilogue, relative to the values it forms
SLOPE = 1.13              # max |d act / dx| of GELU(erf) (1.129); SiLU and quick-GELU peak at 1.100
U32 = 2.0 ** -24


def op_names(ops):
    """Public functions of the ops module (or of the stand-ins patched into it), without its imports."""
    return sorted(n for n, f in vars(ops).items()
                  if not n.startswith("_") and inspect.isfunction(f) and f.__module__ in (ops.__name__, fake_ops.__name__))


# ---------------------------------------------------------------------------------------------------------------------
# comparators: each returns max(err / bar) over the elements (inf for a non-finite output or a wrong shape)
# ---------------------------------------------------------------------------------------------------------------------
def _ratio(out, err, tol):
    if not bool(torch.isfinite(out).all()):
        return float("inf")
    return float((err / tol.clamp_min(1e-300)).max().item()) if err.numel() else 0.0


def ulp_ratio(out, ref, ulps=1.0, slack=None):
    """close_ulps' bar (test_kernel_edges_gpu.py) as a ratio."""
    if out.shape != ref.shape:
        return float("inf")
    err, tol = ulp_err_tol(out, ref, ulps, slack)
    return _ratio(out, err, tol)


def check_ratio(out, ref, rtol, atol):
    """test_kernels_gpu.check's bar (one fp16 rounding of an unrounded reference) as a ratio."""
    if out.shape != ref.shape:
        return float("inf")
    out, ref = out.double(), ref.double()
    return _ratio(out, (out - ref).abs(), atol + rtol * ref.abs() + ref.abs() * 2.0 ** -11)


def exact_ratio(out, ref):
    return 0.0 if out.shape == ref.shape and torch.equal(out, ref) else float("inf")


# ---------------------------------------------------------------------------------------------------------------------
# references: (result, bound arguments) -> max err / bar
# ---------------------------------------------------------------------------------------------------------------------
def _f32(t):
    return None if t is None else t.float()


def _rstd_from_slots(stats, K, eps):
    tot = stats.float().sum(dim=0)
    mean = tot[:, 0] / K
    return torch.rsqrt((tot[:, 1] / K - mean * mean).clamp_min(0) + eps)


def acc_allowance(K):
    """Accumulation allowance of a tensor-core GEMM / conv of depth K, per unit of |A| @ |W|^T."""
    return -(-K // 16) * ACC_STEP


def _act_slack(p, pre, s):
    """The accumulation allowance `s` of the pre-activation `pre` carried through the epilogue's activation."""
    if p["geglu"]:
        a, g = pre.chunk(2, dim=-1)
        sa, sg = s.chunk(2, dim=-1)
        return F.gelu(g).abs() * sa + (a.abs() + sa) * SLOPE * sg
    if p["silu"] or p["gelu"] or p["quick_gelu"]:
        return SLOPE * s
    return s


def ref_linear(res, p):
    x, w, bias, ln = p["x"].double(), p["w"].double(), p["bias"], p["ln"]
    K = x.shape[1]
    kw = dict(rowbias=p["rowbias"], rows_per_group=p["rows_per_group"], geglu=p["geglu"], silu=p["silu"],
              gelu=p["gelu"], quick_gelu=p["quick_gelu"], alpha=p["alpha"])
    resid = 0.0 if p["residual"] is None else p["residual"].double()
    scale = torch.full((x.shape[0], 1), abs(p["alpha"]), dtype=torch.float64, device=x.device)
    if ln is not None:
        scale = scale * _rstd_from_slots(ln[0], K, ln[1]).double()[:, None]
    mag = x.abs() @ w.abs().t()
    acc = x @ w.t()
    pre = acc * scale + (0.0 if bias is None else bias.double())
    s = acc_allowance(K) * mag * scale + EPI * pre.abs()
    if ln is not None:
        var = x.var(dim=1, unbiased=False)
        rel = 0.5 * 3 * K * U32 * x.pow(2).mean(dim=1) / (var + ln[1]) + 2.0 ** -22
        s = s + rel[:, None] * (acc * scale).abs()
    s = _act_slack(p, pre, s)

    def ratio(act):          # act: the epilogue's value before the residual, unrounded fp64
        ref = act + resid
        return ulp_ratio(res, ref, 0.5, s + EPI * (ref.abs() + act.abs()))
    worst = ratio(fake_ops.linear(x, w, bias, ln=ln, **kw))
    if ln is not None:
        # the same GEMM with the true fp64 statistics of the raw rows: rstd * x through the plain path
        rstd64 = torch.rsqrt(x.var(dim=1, unbiased=False) + ln[1])
        worst = max(worst, ratio(fake_ops.linear(x * rstd64[:, None], w, bias, **kw)))
    if p["stats_out"] is not None:
        worst = max(worst, stats_ratio(p["stats_out"], res))
    return worst


def stats_ratio(stats, out):
    """Slot totals of a GEMM's `stats_out` against the fp64 row sum / sum of squares of its stored fp16 output."""
    o = out.double()
    got = stats.double().sum(dim=0)
    n = o.shape[1]
    r1 = _ratio(got, (got[:, 0] - o.sum(1)).abs(), n * U32 * o.abs().sum(1))
    r2 = _ratio(got, (got[:, 1] - o.pow(2).sum(1)).abs(), n * U32 * o.pow(2).sum(1))
    return max(r1, r2)


def ref_conv3x3(res, p):
    sc = p["shortcut"]
    x, w = p["x"].double(), p["w_packed"].double()
    sc64 = None if sc is None else (sc[0].double(), None if sc[1] is None else sc[1].double())
    pre = fake_ops.conv3x3(x, w, p["bias"], rowbias=p["rowbias"], shortcut=sc64, stride=p["stride"], alpha=p["alpha"])
    ref = pre + (0.0 if p["residual"] is None else p["residual"].double())
    sc_abs = None if sc64 is None else tuple(None if t is None else t.abs() for t in sc64)
    mag = fake_ops.conv3x3(x.abs(), w.abs(), stride=p["stride"], alpha=abs(p["alpha"]), shortcut=sc_abs)
    return ulp_ratio(res, ref, 0.5, acc_allowance(w.shape[1]) * mag + EPI * (pre.abs() + ref.abs()))


def ref_attention(res, p):
    q, k, v, B, H, Nq, Nk = (p[n] for n in ("q", "k", "v", "B", "H", "Nq", "Nk"))
    kw = dict(n_ip=p["n_ip"])
    per = max(1, (1 << 29) // (H * Nq * Nk))        # images per slice: <= 2 GiB of fp32 scores
    worst = 0.0
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        rq, rk = slice(b0 * Nq, b1 * Nq), slice(b0 * Nk, b1 * Nk)
        ref = fake_ops.attention(q[rq], k[rk], v[rk], b1 - b0, H, Nq, Nk, ip_scale=p["ip_scale"], **kw)
        mag = fake_ops.attention(q[rq].float(), k[rk].float(), v[rk].float().abs(), b1 - b0, H, Nq, Nk,
                                 ip_scale=abs(p["ip_scale"]), **kw)
        worst = max(worst, ulp_ratio(res[rq], ref, 1.0, 2.0 ** -10 * mag))
    return worst


def ref_groupnorm(res, p):
    ref = fake_ops.groupnorm(p["x0"].float(), p["gamma"], p["beta"], x1=_f32(p["x1"]), groups=p["groups"],
                             eps=p["eps"], silu=p["silu"])
    return check_ratio(res, ref, 2e-3, 2e-3)                        # test_groupnorm_* bar


def ref_layernorm(res, p):
    return check_ratio(res, fake_ops.layernorm(p["x"].float(), p["gamma"], p["beta"], p["eps"]), 2e-3, 2e-3)


def ref_linear_small(res, p):
    ref = fake_ops.linear_small(p["x"].float(), p["w"], p["bias"], act_in=p["act_in"], act_out=p["act_out"],
                                addend=p["addend"], out_scale=p["out_scale"])
    return check_ratio(res, ref, 4e-3, 4e-3)                        # test_linear_small_edges' fp64 bar


def ref_sinusoid(res, p):
    return check_ratio(res, fake_ops.sinusoid(p["t"], p["dim"], p["n"], step=p["step"]), 2e-3, 2e-3)  # test_sinusoid


def ref_softmax_rows_masked_(res, p):
    ref = fake_ops.softmax_rows_masked_(p["x"].float(), p["valid_cols"])
    out, ref = res.double(), ref.double()
    return _ratio(out, (out - ref).abs(), 1e-6 + 2e-3 * ref.abs())    # test_softmax_rows_masked_kernel


def _exact(fn, *names):
    return lambda res, p: exact_ratio(res, fn(*(p[n] for n in names)))


REFERENCES = {
    "linear": ref_linear,
    "conv3x3": ref_conv3x3,
    "attention": ref_attention,
    "groupnorm": ref_groupnorm,
    "layernorm": ref_layernorm,
    "linear_small": ref_linear_small,
    "sinusoid": ref_sinusoid,
    "softmax_rows_masked_": ref_softmax_rows_masked_,
    "upsample2x": _exact(fake_ops.upsample2x, "x"),
    "concat_channels": _exact(fake_ops.concat_channels, "x0", "x1"),
    "im2col3x3_nchw": _exact(fake_ops.im2col3x3_nchw, "x_nchw", "kpad"),
    "nhwc_to_nchw": _exact(fake_ops.nhwc_to_nchw, "x", "C"),
}
IN_PLACE = {"softmax_rows_masked_": "x"}       # op -> the argument it overwrites (and returns)
OUTPUTS = {"out", "stats_out"}                  # written by the op: compared after the call, never snapshotted
NOT_KEYED = {"ws"}                            # persistent scratch: its size does not change what the op computes


# ---------------------------------------------------------------------------------------------------------------------
# the recorder
# ---------------------------------------------------------------------------------------------------------------------
def _sig(v):
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype).replace("torch.", ""))
    if isinstance(v, (tuple, list)):
        return tuple(_sig(e) for e in v)
    return v


def _snapshot(v):
    if isinstance(v, torch.Tensor):
        return v.clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_snapshot(e) for e in v)
    return v


def _label(name, p):
    """Short shape text for the report."""
    def dims(t):
        return "x".join(str(d) for d in t.shape)
    if name == "linear":
        flags = [f for f in ("geglu", "silu", "gelu", "quick_gelu") if p[f]]
        flags += [f for f in ("residual", "rowbias", "ln", "stats_out") if p[f] is not None]
        flags += [] if p["alpha"] == 1.0 else [f"alpha={p['alpha']:g}"]
        return f"{p['x'].shape[0]}x{p['w'].shape[0]}x{p['x'].shape[1]} tile_n={p['tile_n']} {' '.join(flags)}"
    if name == "conv3x3":
        flags = [f for f in ("rowbias", "residual", "shortcut") if p[f] is not None]
        flags += [] if p["alpha"] == 1.0 else [f"alpha={p['alpha']:g}"]
        return f"{dims(p['x'])}->{p['w_packed'].shape[0]} s{p['stride']} {' '.join(flags)}"
    if name == "attention":
        return f"B{p['B']} H{p['H']} {p['Nq']}x{p['Nk']} n_ip={p['n_ip']}"
    if name == "groupnorm":
        c1 = 0 if p["x1"] is None else p["x1"].shape[-1]
        return f"{dims(p['x0'])}+{c1} g{p['groups']}{' silu' if p['silu'] else ''}"
    tensors = [v for v in p.values() if isinstance(v, torch.Tensor)]
    return dims(tensors[0]) if tensors else ""


class Census:
    """Wraps the ops for one forward.  check_all: compare every call (else the first call of each key).  plan: an
    optional (op name, bound arguments) -> hashable hook naming the execution plan, which joins the key."""

    def __init__(self, ops, check_all=True, plan=None, references=REFERENCES):
        self.ops, self.check_all, self.plan, self.references = ops, check_all, plan, references
        self.rows = {}          # key -> {"op", "shape", "plan", "calls", "checked", "worst"}

    def install(self, monkeypatch):
        for name in op_names(self.ops):
            if name not in EXEMPT:
                monkeypatch.setattr(self.ops, name, self._wrap(name, getattr(self.ops, name)))
        return self

    def _wrap(self, name, orig):
        sig = inspect.signature(orig)

        def wrapped(*a, **k):
            ref = self.references.get(name)
            if ref is None:
                raise AssertionError(f"ops.{name} has no census reference (tests/census.py REFERENCES)")
            b = sig.bind(*a, **k)
            b.apply_defaults()
            p = dict(b.arguments)
            plan = None if self.plan is None else self.plan(name, p)
            key = (name, plan) + tuple((n, _sig(v)) for n, v in p.items() if n not in NOT_KEYED)
            row = self.rows.get(key)
            if row is None:
                row = self.rows[key] = {"op": name, "shape": _label(name, p), "plan": plan, "calls": 0, "checked": 0,
                                        "worst": 0.0}
            row["calls"] += 1
            if not (self.check_all or row["checked"] == 0):
                return orig(*a, **k)
            # inputs the call may overwrite: an in-place op's operand, or anything when `out` is given (it may alias)
            snap = dict(p)
            if name in IN_PLACE or p.get("out") is not None:
                snap = {n: (v if n in OUTPUTS else _snapshot(v)) for n, v in p.items()}
            res = orig(*a, **k)
            row["checked"] += 1
            row["worst"] = max(row["worst"], ref(res, snap))
            return res
        wrapped.__wrapped_op__ = orig
        return wrapped

    def failures(self):
        return [r for r in self.rows.values() if r["checked"] and not r["worst"] <= 1.0]

    def report(self, title):
        lines = [f"== census: {title}: {len(self.rows)} keys, {sum(r['calls'] for r in self.rows.values())} calls, "
                 f"{sum(r['checked'] for r in self.rows.values())} checked",
                 f"{'op':<22} {'shape':<58} {'plan':<12} {'calls':>5} {'checked':>7} {'err/bar':>8}"]
        for r in sorted(self.rows.values(), key=lambda r: (r["op"], r["shape"])):
            lines.append(f"{r['op']:<22} {r['shape']:<58} {str(r['plan']):<12} {r['calls']:>5} {r['checked']:>7} "
                         f"{r['worst']:>8.3f}")
        return "\n".join(lines)
