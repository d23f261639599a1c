"""fp16 ulp arithmetic and the ulp comparator shared by the kernel edge tests and the census (tests/census.py)."""
import torch


def ulp16(x):
    a = x.abs().double().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def ulp_err_tol(out, ref, ulps=1.0, slack=None):
    """(|out - ref|, ulps * ulp16(max(|out|, |ref|)) + slack) in fp64: the bar of close_ulps, elementwise."""
    out, ref = out.double(), ref.double()
    tol = ulps * ulp16(torch.maximum(out.abs(), ref.abs()))
    if slack is not None:
        tol = tol + slack
    return (out - ref).abs(), tol


def close_ulps(out, ref, what, ulps=1.0, slack=None):
    """|out - ref| <= ulps * ulp16(max(|out|, |ref|)) (+ slack: the fp32 accumulation-order allowance)."""
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err, tol = ulp_err_tol(out, ref, ulps, slack)
    bad = err > tol
    print(f"[{what}] max_abs_err={err.max().item():.3e} max_err/ulp={(err / ulp16(ref)).max().item():.2f}")
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements beyond {ulps} ulp, "
                           f"max err {err.max().item():.3e}")
