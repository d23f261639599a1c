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
  - `relu` (IH_EPI_RELU, applied after the residual): the reference is relu of the fp64 sum and the slack stays that
    of the sum, because ReLU is 1-Lipschitz (|relu(a) - relu(b)| <= |a - b|); the half ulp is of the stored value;
  the fp64 references of convs with more than 2^28 output elements are computed a slice of images at a time;
* the folded-LayerNorm consumer, against both the slot statistics the kernel reads and the true fp64 statistics of
  its raw rows: plus the error of var = E[x^2] - mean^2 from fp32 sums of K terms (the producer's slots and their
  total; each sum off by at most K 2^-24 of its magnitude, the fp16 squares exact in fp32), 3 K 2^-24 E[x^2] /
  (var + eps) relative on var, half of it on rstd, plus 2^-22 for rsqrtf;
* `stats_out` slots: their totals against the row sums of the stored fp16 output in fp64, within N 2^-24 sum|x|
  (resp. sum x^2): any fp32 summation order of N terms;
* attention: P is packed to fp16 before the PV MMA (half an fp16 ulp of every p) and exp / the score sums in fp32 stay
  below another half: 1 ulp + 2^-10 * (P @ |V|), the IP part weighted by |ip_scale|;
* norms, linear_small, sinusoid, masked softmax: the bars of their existing kernel tests, against unrounded fp32;
* conv3x3_down (the VAE encoder's bottom/right-padded stride-2 conv, conv_impl on the same wgmma main loop): the
  conv3x3 bar with K = 9 Cin, against F.pad(x, (0, 1, 0, 1)) and a stride-2, pad-0 conv in fp64;
* conv3x3_small (one thread per output, a sequential fp32 fmaf over the 9 Cin products in tap order, + bias, SiLU as
  acc / (1 + __expf(-acc)), one fp16 rounding), against fp64: half an ulp, plus (9 Cin + 1) 2^-24 (conv |x| * |w| + |b|)
  for the 9 Cin fma roundings and the bias add (round-to-nearest loses at most 2^-24 of a running sum, which never
  exceeds the magnitude), times SLOPE under SiLU, plus EPI |out| for __expf and the divide (a relative error e of
  __expf moves SiLU by at most e |SiLU|);
* attention_generic (fp32 scores by a sequential fma over dqk, times scale; fp32 softmax with __expf; fp32 PV by a
  sequential fma over the live keys; times 1 / sum; one fp16 rounding), against fp64 with the causal mask: half an
  ulp, plus (P @ |V|) times
  - 2 max_j ds_j, the score error ds_j = (dqk + 1) 2^-24 (|q| . |k_j|) scale carried through the softmax (a score
    move ds_j changes p_j by a factor within exp(+-2 max ds)),
  - 2 (2^-21 + 2^-24 max_j |s_j - s_max|) for __expf (ex2.approx and the rounding of its scaled argument),
  - (2 Nk + 3) 2^-24 for the two fp32 sums of Nk terms, 1 / sum and the final product;
* attention_small (fp32 q . k rounded to fp16, divided by the fp32 scale, rounded to fp16 again -- both the
  reference's rounding points, attention_processor.py:45 --; fp32 softmax with __expf; each p stored as fp16 before
  the fp32 PV): the reference takes the same two fp16 roundings of the fp64 dot product.  The kernel's fp32 dot product
  may round to the neighbouring fp16 score, so every score may be 1 fp16 ulp off: with d = max_j ulp16(s_j) each p_j
  moves by a factor within exp(+-2d), and as sum p_j = 1 on both sides that costs (e^{2d} - 1) (P @ |V - out|).  Then
  the fp16 store of p (2^-11 p_j, or 2^-25 below the fp16 normal range) and the fp32 arithmetic before it (__expf and the
  sum, as for attention_generic), over P @ |V| resp. sum |V|; plus (Nk + 1) 2^-24 (P @ |V|) for the PV sum, and half an
  ulp of the output;
* embed_tokens, add_bcast: bit-exact against (a.float() + b.float()).half() (embed_tokens with the ids clamped to the
  vocabulary as the kernel clamps them): fp32 carries at least 2 * 11 + 2 significant bits, so rounding the exact sum
  of two fp16 values first to fp32 and then to fp16 gives the same fp16 value as rounding it once;
* mean_tokens (a sequential fp32 sum of n terms, times the fp32 reciprocal of n, one fp16 rounding), against fp64:
  half an ulp, plus n 2^-24 mean|x| for the sum, plus 2 2^-24 |out| for the reciprocal and the product;
* resize_patchify (area average in fp32, [0, 1], (v - mean) / std), against oracle.clip_ref.resize_patchify_ref in
  fp64, per element: the pixel-boundary products oy * fy round twice (fy, then the product), so each boundary moves by
  at most Hin 2^-23; only the two edge rows and columns of a window carry a boundary, so the area-weighted average
  moves by at most 2 max|x| (2 fx Hin 2^-23 + 2 fy Win 2^-23) / (fy fx) = max|x| S 2^-20, plus 2 max|x| 2^-24 for the
  wy * wx products and 2 n_px 2^-24 max|x| for the two fma sums over the window's n_px pixels, 2^-24 for the divide;
  then * 0.5 + 0.5, - mean and / std add four fp32 roundings of values below 1 + max|x| and the / std multiplies the
  error by up to 1 / min(std) = 3.8; plus half an ulp of the output;
* im2col3x3_nchw_cat, controlnet_add_residuals(_multi): bit-exact against the stand-ins (tests/fake_ops_inpaint9.py,
  tests/fake_ops_controlnet.py, tests/fake_ops_multi_controlnet.py), which round where the kernels round.  The two
  injection ops add into `skips` in place: the reference applies the stand-in to a snapshot taken before the call and
  compares every skip tensor after it, rows outside the injected window included;
* vae_posterior_noise: the bar of test_img2img_gpu.py::test_posterior_noise_kernel, 1 fp16 ulp against
  img2img_ref.posterior_noise_ref (the same rounding points; the fp32 exp may differ in the last bit), and overflow to
  inf at the same elements.

The scheduler step kernels and the model-input scaling are not model ops: STEP_KERNELS names the bit-exact test that
checks each at SDXL bucket latent sizes.

A reference that ignores one of its op's arguments would pass a kernel that ignores it too.  So each reference reads
its arguments through a dict that records the keys read, and `Census.unread()` lists every (op, argument) of the
calls checked that the reference never read and that UNREAD does not excuse.
"""
import inspect
import math

import torch
import torch.nn.functional as F

import fake_ops
import fake_ops_controlnet
import fake_ops_img2img
import fake_ops_inpaint9
import fake_ops_multi_controlnet
from fp16_ulps import ulp16, ulp_err_tol

EXEMPT = {"prefetch_next", "fold_layernorm", "pack_conv3x3_weight", "workspace_generation", "launch_count",
          "launch_count_reset"}
STEP_KERNELS = {       # op -> the test that checks it bit-exactly at SDXL bucket latent sizes
    "euler_cfg_step": "test_kernels_gpu.py::test_euler_cfg_step",
    "euler_step": "test_kernels_gpu.py::test_euler_step_ex",
    "euler_inpaint_step": "test_inpaint_gpu.py::test_euler_inpaint_step_kernel",
    "dpm_solver_step": "test_dpm_gpu.py::test_dpm_solver_step_kernel",
    "euler_ancestral_step": "test_euler_a_gpu.py::test_euler_ancestral_step_kernel",
    "scale_model_input": "test_kernel_edges_gpu.py::test_scale_model_input_entry",
    "euler_ancestral_scale_input": "test_euler_a_gpu.py::test_first_input_equals_torch_scale_model_input",
}
ACC_STEP = 2.0 ** -23     # one rounding of the fp32 accumulator per k16 MMA step, relative to |A| @ |W|^T
EPI = 2.0 ** -21          # the fp32 epilogue, relative to the values it forms
SLOPE = 1.13              # max |d act / dx| of GELU(erf) (1.129); SiLU and quick-GELU peak at 1.100
U32 = 2.0 ** -24


def _is_stand_in(module_name):
    return module_name.rsplit(".", 1)[-1].startswith("fake_ops")     # tests/fake_ops.py and every tests/fake_ops_*.py


def op_names(ops):
    """Public functions of the ops module (or of the stand-ins patched into it), without its imports."""
    return sorted(n for n, f in vars(ops).items()
                  if not n.startswith("_") and inspect.isfunction(f)
                  and (f.__module__ == ops.__name__ or _is_stand_in(f.__module__)))


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
    x, w, bias, ln, relu = p["x"].double(), p["w"].double(), p["bias"], p["ln"], p["relu"]
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
        tot = act + resid
        return ulp_ratio(res, torch.relu(tot) if relu else tot, 0.5, s + EPI * (tot.abs() + act.abs()))
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
    sc, rowbias, residual, stride, alpha, relu = (p[n] for n in ("shortcut", "rowbias", "residual", "stride", "alpha",
                                                                "relu"))
    w = p["w_packed"].double()
    B = p["x"].shape[0]
    per = max(1, (1 << 28) // res[0].numel())        # images per slice: <= 2 GiB per fp64 output-sized tensor
    worst = 0.0
    for b0 in range(0, B, per):
        i = slice(b0, min(B, b0 + per))
        x = p["x"][i].double()
        sc64 = None if sc is None else (sc[0][i].double(), None if sc[1] is None else sc[1][i].double())
        pre = fake_ops.conv3x3(x, w, p["bias"], rowbias=None if rowbias is None else rowbias[i], shortcut=sc64,
                               stride=stride, alpha=alpha)
        tot = pre + (0.0 if residual is None else residual[i].double())
        sc_abs = None if sc64 is None else tuple(None if t is None else t.abs() for t in sc64)
        mag = fake_ops.conv3x3(x.abs(), w.abs(), stride=stride, alpha=abs(alpha), shortcut=sc_abs)
        worst = max(worst, ulp_ratio(res[i], torch.relu(tot) if relu else tot, 0.5,
                                     acc_allowance(w.shape[1]) * mag + EPI * (pre.abs() + tot.abs())))
    return worst


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


def _w4(w_packed, Cin):
    """Tap-major [Cout, 9 Cin] -> OIHW [Cout, Cin, 3, 3] in fp64."""
    return w_packed.double().reshape(w_packed.shape[0], 3, 3, Cin).permute(0, 3, 1, 2)


def ref_conv3x3_down(res, p):
    x = p["x"].double()
    w = _w4(p["w_packed"], x.shape[-1])

    def conv(x, w, alpha):
        return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1)), w, stride=2).permute(0, 2, 3, 1) * alpha
    ref = conv(x, w, p["alpha"]) + (0.0 if p["bias"] is None else p["bias"].double())
    mag = conv(x.abs(), w.abs(), abs(p["alpha"]))
    return ulp_ratio(res, ref, 0.5, acc_allowance(9 * x.shape[-1]) * mag + 2 * EPI * ref.abs())


def ref_conv3x3_small(res, p):
    x = p["x"].double()
    x = x if p["nchw"] else x.permute(0, 3, 1, 2)
    Cin = x.shape[1]
    w = _w4(p["w_packed"], Cin)
    b = None if p["bias"] is None else p["bias"].double()
    pre = F.conv2d(x, w, b, stride=p["stride"], padding=1)
    s = (9 * Cin + 1) * U32 * F.conv2d(x.abs(), w.abs(), None if b is None else b.abs(), stride=p["stride"], padding=1)
    ref = pre
    if p["silu"]:
        ref = F.silu(pre)
        s = SLOPE * s + EPI * ref.abs()
    return ulp_ratio(res, ref.permute(0, 2, 3, 1), 0.5, s.permute(0, 2, 3, 1))


def _heads(t, B, N, H, d):
    return t[:, :H * d].double().reshape(B, N, H, d).transpose(1, 2)


def _flat(t):
    B, H, N, d = t.shape
    return t.transpose(1, 2).reshape(B * N, H * d)


def ref_attention_generic(res, p):
    B, H, Nq, Nk, dqk, dv, scale = (p[n] for n in ("B", "H", "Nq", "Nk", "dqk", "dv", "scale"))
    q, k, v = _heads(p["q"], B, Nq, H, dqk), _heads(p["k"], B, Nk, H, dqk), _heads(p["v"], B, Nk, H, dv)
    s = q @ k.transpose(-1, -2) * scale
    smag = q.abs() @ k.abs().transpose(-1, -2) * abs(scale)
    live = torch.ones(Nq, Nk, dtype=torch.bool, device=s.device)
    if p["causal"]:
        live = live.tril(Nk - Nq)
    s = s.masked_fill(~live, float("-inf"))
    P = s.softmax(-1)
    ds = (dqk + 1) * U32 * smag.masked_fill(~live, 0).amax(-1, keepdim=True)
    spread = (s.amax(-1, keepdim=True) - s).masked_fill(~live, 0).amax(-1, keepdim=True)
    rel = 2 * ds + 2 * (2.0 ** -21 + U32 * spread) + (2 * Nk + 3) * U32
    return ulp_ratio(res, _flat(P @ v), 0.5, _flat(rel * (P @ v.abs())))


def ref_attention_small(res, p):
    B, H, Nq, Nk, dqk, dv = (p[n] for n in ("B", "H", "Nq", "Nk", "dqk", "dv"))
    q, k, v = _heads(p["q"], B, Nq, H, dqk), _heads(p["k"], B, Nk, H, dqk), _heads(p["v"], B, Nk, H, dv)
    scale32 = float(torch.tensor(p["scale"], dtype=torch.float32))        # the kernel divides by the fp32 value
    qk16 = (q @ k.transpose(-1, -2)).half().double()
    s16 = (qk16 / scale32).half().double()
    P = s16.softmax(-1)
    out = P @ v
    # a neighbouring fp16 q.k moves the quotient by ulp16(q.k) / scale before its own rounding
    d = (ulp16(qk16) / scale32 + ulp16(s16)).amax(-1, keepdim=True)
    grow = torch.exp(2 * d)
    spread = (s16.amax(-1, keepdim=True) - s16).amax(-1, keepdim=True)
    pre = 2.0 ** -21 + U32 * spread + (Nk + 2) * U32                      # __expf, the fp32 sum, 1 / sum, p * inv
    pv = grow * (P @ v.abs())
    centred = (P[..., None] * (v[:, :, None] - out[:, :, :, None]).abs()).sum(-2)      # sum_j p_ij |v_j - out_i|
    slack = ((grow - 1) * centred + (2.0 ** -11 + pre + (Nk + 1) * U32) * pv
             + 2.0 ** -25 * v.abs().sum(-2, keepdim=True))
    return ulp_ratio(res, _flat(out), 0.5, _flat(slack))


def ref_embed_tokens(res, p):
    ids, tok, pos = p["ids"], p["tok_emb"], p["pos_emb"]
    B, T = ids.shape
    rows = tok[ids.long().clamp(0, tok.shape[0] - 1)]
    return exact_ratio(res, (rows.float() + pos[:T].float()[None]).to(tok.dtype).reshape(B * T, -1))


def ref_add_bcast(res, p):
    a, b = p["a"], p["b"]
    return exact_ratio(res, (a.float().reshape(-1, b.numel()) + b.float().reshape(1, -1)).to(a.dtype).reshape(a.shape))


def ref_mean_tokens(res, p):
    x = p["x"].double()
    ref = x.mean(dim=1)
    return ulp_ratio(res, ref, 0.5, x.shape[1] * U32 * x.abs().mean(dim=1) + 2 * U32 * ref.abs())


def ref_resize_patchify(res, p):
    from oracle.clip_ref import resize_patchify_ref
    img, S = p["img"], p["size"]
    _, _, Hin, Win = img.shape
    ref = resize_patchify_ref(img.cpu().double(), S, p["patch"], p["kpad"], p["mean"], p["std"], dtype=torch.float64)
    A = float(img.abs().max())
    n_px = (math.ceil(Hin / S) + 2) * (math.ceil(Win / S) + 2)
    d_avg = A * (S * 2.0 ** -20 + 2 * U32 + 2 * n_px * U32 + U32)
    d = (0.5 * d_avg + 4 * U32 * (1 + A)) / min(float(s) for s in p["std"])
    return ulp_ratio(res.cpu(), ref, 0.5, d + U32 * ref.abs())


def _injection_ratio(res, p, inject):
    """Every skip tensor after an in-place injection against the stand-in applied to the pre-call snapshot."""
    want = [s.clone() for s in p["skips"]]
    inject(want)
    if len(res) != len(want):
        return float("inf")
    return max(exact_ratio(r, w) for r, w in zip(res, want))


def ref_controlnet_add_residuals(res, p):
    return _injection_ratio(res, p, lambda sk: fake_ops_controlnet.controlnet_add_residuals(
        sk, p["residuals"], p["scale"], p["skip_row0s"]))


def ref_controlnet_add_residuals_multi(res, p):
    return _injection_ratio(res, p, lambda sk: fake_ops_multi_controlnet.controlnet_add_residuals_multi(
        sk, p["residuals_per_net"], p["scales_per_net"], p["skip_row0s"]))


def ref_vae_posterior_noise(res, p):
    ref = fake_ops_img2img.vae_posterior_noise(p["moments"], p["eps"], p["noise"], p["channels"], p["scaling_factor"],
                                               p["sigma"])
    fin = torch.isfinite(ref)
    if res.shape != ref.shape or not torch.equal(torch.isfinite(res), fin) or not torch.equal(res[~fin], ref[~fin]):
        return float("inf")
    return ulp_ratio(res[fin], ref[fin], 1.0)                              # test_posterior_noise_kernel's bar


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
    "conv3x3_down": ref_conv3x3_down,
    "conv3x3_small": ref_conv3x3_small,
    "attention_generic": ref_attention_generic,
    "attention_small": ref_attention_small,
    "embed_tokens": ref_embed_tokens,
    "add_bcast": ref_add_bcast,
    "mean_tokens": ref_mean_tokens,
    "resize_patchify": ref_resize_patchify,
    "im2col3x3_nchw_cat": _exact(fake_ops_inpaint9.im2col3x3_nchw_cat, "x0", "x1", "kpad"),
    "controlnet_add_residuals": ref_controlnet_add_residuals,
    "controlnet_add_residuals_multi": ref_controlnet_add_residuals_multi,
    "vae_posterior_noise": ref_vae_posterior_noise,
}
# op -> the argument it overwrites: an op that returns it gets it back; for one that returns None (the ControlNet
# injections) the reference receives the argument itself, after the call, as the result
IN_PLACE = {"softmax_rows_masked_": "x", "controlnet_add_residuals": "skips", "controlnet_add_residuals_multi": "skips"}
OUTPUTS = {"out", "stats_out"}                  # written by the op: compared after the call, never snapshotted
NOT_KEYED = {"ws"}                            # persistent scratch: its size does not change what the op computes
UNREAD = {             # arguments a reference may leave unread, and why; any other unread argument fails the census
    "out": "the destination: the reference compares what the op wrote there (or returned)",
    "tile_n": "GEMM / conv tile width: every output still sums its own K products in one fp32 accumulator, so the bar "
              "holds for every width; the census key records it",
    "kv_split": "attention work split: the bar of the unsplit softmax covers the split-and-merge (test_kernels_gpu.py"
                "::test_attention_kv_split checks the two plans against each other)",
    "ws": "GroupNorm's persistent scratch, not an input",
}


class _Reads(dict):
    """Bound arguments that record which keys a reference reads."""

    def __init__(self, p):
        super().__init__(p)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        self.read.add(k)
        return super().get(k, default)


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
        flags = [f for f in ("geglu", "silu", "gelu", "quick_gelu", "relu") if p[f]]
        flags += [f for f in ("residual", "rowbias", "ln", "stats_out") if p[f] is not None]
        flags += [] if p["alpha"] == 1.0 else [f"alpha={p['alpha']:g}"]
        return f"{p['x'].shape[0]}x{p['w'].shape[0]}x{p['x'].shape[1]} tile_n={p['tile_n']} {' '.join(flags)}"
    if name == "conv3x3":
        flags = [f for f in ("rowbias", "residual", "shortcut") if p[f] is not None]
        flags += ["relu"] if p["relu"] else []
        flags += [] if p["alpha"] == 1.0 else [f"alpha={p['alpha']:g}"]
        return f"{dims(p['x'])}->{p['w_packed'].shape[0]} s{p['stride']} {' '.join(flags)}"
    if name == "attention":
        return f"B{p['B']} H{p['H']} {p['Nq']}x{p['Nk']} n_ip={p['n_ip']}"
    if name == "groupnorm":
        c1 = 0 if p["x1"] is None else p["x1"].shape[-1]
        return f"{dims(p['x0'])}+{c1} g{p['groups']}{' silu' if p['silu'] else ''}"
    if name in ("attention_generic", "attention_small"):
        causal = " causal" if p.get("causal") else ""
        return f"B{p['B']} H{p['H']} {p['Nq']}x{p['Nk']} d{p['dqk']}/{p['dv']}{causal}"
    if name == "conv3x3_small":
        return (f"{dims(p['x'])}{' nchw' if p['nchw'] else ''}->{p['w_packed'].shape[0]} s{p['stride']}"
                f"{' silu' if p['silu'] else ''}")
    if name == "conv3x3_down":
        return f"{dims(p['x'])}->{p['w_packed'].shape[0]}" + ("" if p["alpha"] == 1.0 else f" alpha={p['alpha']:g}")
    if name == "resize_patchify":
        return f"{dims(p['img'])}->{p['size']}"
    if name == "vae_posterior_noise":
        return f"moments {dims(p['moments'])} eps {dims(p['eps'])} {p['eps'].dtype} noise {dims(p['noise'])}"
    if name in IN_PLACE and name != "softmax_rows_masked_":
        nets = f" K{len(p['residuals_per_net'])}" if "residuals_per_net" in p else ""
        return f"{len(p['skips'])} skips {dims(p['skips'][0])} row0 {p['skip_row0s'][0]}{nets}"
    tensors = [v for v in p.values() if isinstance(v, torch.Tensor)]
    return dims(tensors[0]) if tensors else ""


class Census:
    """Wraps the ops for one forward.  check_all: compare every call (else the first call of each key).  plan: an
    optional (op name, bound arguments) -> hashable hook naming the execution plan, which joins the key."""

    def __init__(self, ops, check_all=True, plan=None, references=REFERENCES):
        self.ops, self.check_all, self.plan, self.references = ops, check_all, plan, references
        self.rows = {}          # key -> {"op", "shape", "plan", "calls", "checked", "worst"}
        self.args = {}          # op -> (arguments of its checked calls, the ones its reference read)

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
            got = p[IN_PLACE[name]] if res is None and name in IN_PLACE else res
            reads = _Reads(snap)
            row["worst"] = max(row["worst"], ref(got, reads))
            have, read = self.args.setdefault(name, (set(), set()))
            have.update(p)
            read.update(reads.read)
            return res
        wrapped.__wrapped_op__ = orig
        return wrapped

    def failures(self):
        return [r for r in self.rows.values() if r["checked"] and not r["worst"] <= 1.0]

    def unread(self):
        """"op(argument)" for every argument of a checked call that the op's reference never read, except UNREAD."""
        return sorted(f"{op}({a})" for op, (have, read) in self.args.items() for a in have - read - set(UNREAD))

    def report(self, title):
        lines = [f"== census: {title}: {len(self.rows)} keys, {sum(r['calls'] for r in self.rows.values())} calls, "
                 f"{sum(r['checked'] for r in self.rows.values())} checked",
                 f"{'op':<22} {'shape':<58} {'plan':<12} {'calls':>5} {'checked':>7} {'err/bar':>8}"]
        for r in sorted(self.rows.values(), key=lambda r: (r["op"], r["shape"])):
            lines.append(f"{r['op']:<22} {r['shape']:<58} {str(r['plan']):<12} {r['calls']:>5} {r['checked']:>7} "
                         f"{r['worst']:>8.3f}")
        return "\n".join(lines)
