"""The census plumbing of test_unet_census_gpu.py without a GPU: the TINY UNet at a non-square latent on the stand-in
ops (tests/fake_ops.py) runs under the recorder, every op it calls has a reference that reads every argument of the
op, an op without one fails the run, the dedupe key checks each distinct call once, and the comparators reject an
output one element of which is 2 fp16 ulps off."""
import pytest
import torch

import census
import fake_ops
from test_wiring_cpu import _build, patched  # noqa: F401  (fixture)


def _forward(lat_h=16, lat_w=24):
    from imagharmony_b200.config import TINY
    native, _ = _build(TINY, 0)
    g = torch.Generator("cpu").manual_seed(3)
    B = 2
    sample = torch.randn(B, 4, lat_h, lat_w, generator=g)
    ehs = torch.randn(B, 77 + TINY.num_ip_tokens, TINY.cross_attention_dim, generator=g)
    te = torch.randn(B, TINY.pooled_embed_dim, generator=g)
    tid = torch.tensor([[lat_h * 8., lat_w * 8., 0., 0., lat_h * 8., lat_w * 8.]] * B)
    with torch.no_grad():
        return native(sample, torch.full((B,), 321.0), ehs, te, tid)


@pytest.mark.parametrize("check_all", [True, False])
def test_every_op_of_the_forward_has_a_reference(patched, monkeypatch, check_all):  # noqa: F811
    from imagharmony_b200 import ops
    c = census.Census(ops, check_all=check_all).install(monkeypatch)
    out = _forward()
    assert out.shape == (2, 4, 16, 24)
    print(c.report("TINY 16x24"))
    called = {r["op"] for r in c.rows.values()}
    assert {"linear", "conv3x3", "attention", "groupnorm", "linear_small", "sinusoid", "upsample2x", "im2col3x3_nchw",
            "nhwc_to_nchw"} <= called <= set(census.REFERENCES)
    assert not c.unread(), f"arguments no reference reads: {c.unread()}"
    assert not c.failures(), c.report("TINY 16x24")
    calls, checked = sum(r["calls"] for r in c.rows.values()), sum(r["checked"] for r in c.rows.values())
    assert checked == (calls if check_all else len(c.rows))
    assert calls > len(c.rows)          # repeated shapes share a key
    # the folded LayerNorm consumers and the statistics producers are among the checked calls
    assert any("ln" in r["shape"].split() for r in c.rows.values() if r["op"] == "linear")
    assert any("stats_out" in r["shape"].split() for r in c.rows.values() if r["op"] == "linear")


def test_an_op_without_a_reference_fails_the_census(patched, monkeypatch):  # noqa: F811
    from imagharmony_b200 import ops
    refs = {k: v for k, v in census.REFERENCES.items() if k != "upsample2x"}
    census.Census(ops, references=refs).install(monkeypatch)
    with pytest.raises(AssertionError, match="ops.upsample2x has no census reference"):
        _forward()


def test_only_host_helpers_are_exempt():
    from imagharmony_b200 import ops
    names = census.op_names(ops)
    assert census.EXEMPT <= set(names)
    assert {"linear", "attention", "euler_step", "controlnet_add_residuals"} <= set(names)
    assert "check" not in names                     # imported from _lib, not an op


def _nudge(t, ulps=2):
    """t with its largest element moved `ulps` fp16 steps toward zero (inside its binade: the step stays one ulp)."""
    t = t.clone()
    flat = t.view(-1)
    i = int(flat.abs().argmax())
    v = flat[i:i + 1]
    for _ in range(ulps):
        v = torch.nextafter(v, torch.zeros_like(v))
    flat[i] = v[0]
    return t


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator("cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half()


def test_comparators_reject_two_ulps():
    x, w, b = _rnd(40, 128, seed=1), _rnd(72, 128, scale=128 ** -0.5, seed=2), _rnd(72, seed=3)
    p = dict(x=x, w=w, bias=b, residual=None, rowbias=None, rows_per_group=0, geglu=False, silu=False, gelu=False,
             out=None, tile_n=0, ln=None, stats_out=None, quick_gelu=False, alpha=1.0, relu=False)
    good = fake_ops.linear(x, w, b)
    assert census.ref_linear(good, p) <= 1.0
    assert census.ref_linear(_nudge(good), p) > 1.0

    xc, wc = _rnd(2, 6, 10, 64, seed=4), _rnd(96, 9 * 64, scale=(9 * 64) ** -0.5, seed=5)
    pc = dict(x=xc, w_packed=wc, bias=None, rowbias=None, residual=None, stride=2, out=None, tile_n=0, alpha=1.0,
              shortcut=None, relu=False)
    good = fake_ops.conv3x3(xc, wc, stride=2)
    assert census.ref_conv3x3(good, pc) <= 1.0
    assert census.ref_conv3x3(_nudge(good), pc) > 1.0

    # attention's bar adds 2^-10 (P @ |V|): with V >= 0, P @ |V| is the output itself and the bar stays below 3 ulps
    B, H, N, n_ip = 2, 2, 40, 4
    q, k, v = _rnd(B * N, H * 64, seed=6), _rnd(B * N, H * 64, seed=7), _rnd(B * N, H * 64, seed=8).abs()
    pa = dict(q=q, k=k, v=v, B=B, H=H, Nq=N, Nk=N, n_ip=n_ip, ip_scale=0.6, out=None, kv_split=True)
    good = fake_ops.attention(q, k, v, B, H, N, N, n_ip=n_ip, ip_scale=0.6)
    assert census.ref_attention(good, pa) <= 1.0
    assert census.ref_attention(_nudge(good, 2), pa) <= 1.0 < census.ref_attention(_nudge(good, 3), pa)

    assert census.exact_ratio(good, good.clone()) == 0.0
    assert census.exact_ratio(_nudge(good, 1), good) == float("inf")
