"""Planted-marker parity of the reducing kernels (tests/planted.py): GroupNorm (fused and two-kernel), the attention
key mask, online softmax and KV-split merge (both multi-block kernels, both split policies, the two-segment
text | image-prompt path), LayerNorm, the masked row softmax and the guidance-rescale std of the four step kernels.
The inputs make every fp32 partial sum exact and the result dominated by a few markers on the kernels' partition
seams, so one element lost, counted twice or credited to the wrong image, row, group, head or key block fails the
ulp-level bar; test_planted_cpu.py shows by how much."""
import os
import subprocess
import sys

import pytest
import torch

import planted as P
from fp16_ulps import close_ulps
from imagharmony_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# IH_GN_FUSED is read once per process; test_groupnorm_planted_two_kernel_path re-runs the GroupNorm cases in a child
GN_TWO_KERNEL = os.environ.get("IH_GN_FUSED", "1")[:1] == "0"
STEP_BUCKETS = [(104, 152), (80, 192), (96, 168), (128, 128)]


@pytest.fixture(scope="module")
def ops():
    from imagharmony_b200 import ops as _ops
    return _ops


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def report(what, worst):
    print(f"[planted {what}] max err/bar {worst:.3f}")
    assert worst <= 1.0, f"{what}: err / bar {worst:.3f}"


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------
def _groupnorm_planted(ops, B, HW, C0, C1, groups, silu, scale):
    """Every launch of the case on the one shared workspace, each with its own marker set."""
    C = C0 + C1
    eps = 1e-5 if scale == 1 else 1e-6 * scale * scale          # the VAE's 2^-7-scaled stream
    cover = P.gn_cover_rows(B, HW, C, sms())
    n = P.gn_launches(B, HW, C, groups, sms())
    gamma, beta = (t.cuda() for t in P.gn_params(C))
    worst = 0.0
    for L in range(n):
        mk = P.gn_markers(B, HW, C, groups, L, n, cover, C0 if C1 else None)
        x = P.gn_build(B, HW, C, mk, scale, device="cuda")
        x0 = x[..., :C0].contiguous().view(B, HW, 1, C0)
        x1 = x[..., C0:].contiguous().view(B, HW, 1, C1) if C1 else None
        n0 = ops.launch_count()
        out = ops.groupnorm(x0, gamma, beta, x1=x1, groups=groups, eps=eps, silu=silu)
        assert ops.launch_count() - n0 == (2 if GN_TWO_KERNEL else 1)
        r = P.gn_check_ratio(out.view(B, HW, C), x, gamma, beta, groups, eps, silu)
        assert r <= 1.0, f"launch {L} of {n}: err / bar {r:.3f}"
        worst = max(worst, r)
        del x, x0, x1, out
    report(f"groupnorm B{B} HW{HW} C{C0}+{C1} g{groups} silu{silu} x{n}{' two-kernel' if GN_TWO_KERNEL else ''}",
           worst)


@pytest.mark.parametrize("B,HW,C0,C1,groups,silu,scale", P.GN_CASES)
def test_groupnorm_planted(ops, B, HW, C0, C1, groups, silu, scale):
    _groupnorm_planted(ops, B, HW, C0, C1, groups, silu, scale)


@pytest.mark.skipif(GN_TWO_KERNEL, reason="this process already runs the two-kernel path")
def test_groupnorm_planted_two_kernel_path():
    """The planted GroupNorm cases once more with IH_GN_FUSED=0 (statistics kernel + apply kernel), in a child."""
    env = dict(os.environ, IH_GN_FUSED="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.abspath(__file__), "-k", "groupnorm and not two_kernel"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    print("\n".join(line for line in r.stdout.splitlines() if "[planted" in line or "passed" in line))
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-2000:]


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [1, 5])
@pytest.mark.parametrize("C", [8, 264, 640, 1280, 2048, 5120, 8192])
def test_layernorm_planted(ops, C, extra):
    rows = P.ln_rows(C, extra)
    g, b = (t.cuda() for t in P.ln_params(C))
    worst = 0.0
    for seed in range(3):
        x = P.ln_build(rows, C, seed=seed, device="cuda")
        out = ops.layernorm(x, g, b, 1e-5)
        ref, slack = P.ln_reference(x, g, b, 1e-5)
        worst = max(worst, P.ratio(out, ref, 1.0, slack))
    report(f"layernorm {rows}x{C}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# masked row softmax
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [168, 1024, 4096, 16384, 32768])
def test_softmax_rows_masked_planted(ops, cols):
    """Tied maxima at the vector, thread and loop seams and at valid - 1; the padding columns start at +60000, must not
    be read and must be written as 0; the columns past `cols` of the wider row stride are not touched."""
    worst = 0.0
    for valid in sorted({1, 7, 9, cols - 1, cols}):
        buf, x = P.smx_build(24, cols, valid, cols + 64, device="cuda")
        ref = P.smx_reference(x, valid)
        ops.softmax_rows_masked_(x, valid)
        assert bool((x[:, valid:] == 0).all()), f"valid {valid}: padding columns not written as 0"
        assert bool((buf[:, cols:] == P.SMX_PAD).all()), f"valid {valid}: wrote past the row"
        worst = max(worst, P.ratio(x, ref))
    report(f"softmax_rows_masked {cols}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _attention_variants(ops, views, B, H, Nq, Nk, ref, slack, what):
    """Both multi-block kernels x both KV-split policies x with / without the workspace, against one reference."""
    lib = _lib.load()
    q, k, v = views
    worst = 0.0
    try:
        for kernel in (0, 1):
            lib.ih_attention_set_kernel(kernel)
            for policy in (0, 1):
                lib.ih_attention_set_split_policy(policy)
                if policy == 1:
                    assert lib.ih_attention_workspace_bytes(B, H, Nq, Nk, 0) > 0, f"{what}: no KV split planned"
                for kv_split in (True, False):
                    out = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=kv_split)
                    r = P.ratio(out, ref, 1.0, slack)
                    assert r <= 1.0, f"{what} kernel {kernel} policy {policy} kv_split {kv_split}: err / bar {r:.3f}"
                    worst = max(worst, r)
    finally:
        lib.ih_attention_set_kernel(0)
        lib.ih_attention_set_split_policy(0)
    report(what, worst)


@pytest.mark.parametrize("merge", [False, True])
@pytest.mark.parametrize("B,H,Nq,Nk", [
    (2, 2, 300, 129), (2, 2, 200, 255), (2, 2, 333, 257), (2, 2, 500, 576), (2, 2, 250, 988), (1, 2, 300, 3952),
    (1, 2, 200, 4096), (2, 1, 300, 4097),
    (2, 10, 4096, 4096), (2, 20, 1024, 1024),          # SDXL self-attention at 1024^2
])
def test_attention_planted(ops, B, H, Nq, Nk, merge):
    """merge=False: 1-6 tied markers per row at key 0, both sides of block boundaries and Nk - 1, a zero-filled
    padding key 4 nats above them; merge=True: two markers one nat apart in different blocks, in both orders.
    Strided views whose outside columns, like the neighbouring batch and head, would dominate any row reading them."""
    if merge and H > 2:
        pytest.skip("the merge case runs at the small shapes")
    _, views = P.att_build(B, H, Nq, Nk, pad=8, merge=merge, device="cuda")
    ref, slack = P.att_reference(*views, B, H, Nq, Nk)
    _attention_variants(ops, views, B, H, Nq, Nk, ref, slack, f"attention B{B} H{H} {Nq}x{Nk} merge{merge}")


@pytest.mark.parametrize("Nk", [33, 81, 93, 128])
def test_attention_two_segment_planted(ops, Nk):
    """Nk <= 128: markers at n_text - 1, n_text and Nk - 1; n_ip in {0, 1, 4, 16, Nk - 1}, ip_scale in {0, 0.6, 1};
    with ip_scale 0 the image-prompt keys contribute exactly nothing."""
    B, H, Nq = 2, 4, 300
    worst = 0.0
    for n_ip in sorted({0, 1, 4, 16, Nk - 1}):
        _, (q, k, v) = P.att_build(B, H, Nq, Nk, pad=8, n_ip=n_ip, device="cuda")
        for ip_scale in (0.0, 0.6, 1.0):
            out = ops.attention(q, k, v, B, H, Nq, Nk, n_ip=n_ip, ip_scale=ip_scale)
            ref, slack = P.att_reference(q, k, v, B, H, Nq, Nk, n_ip, ip_scale)
            r = P.ratio(out, ref, 1.0, slack)
            assert r <= 1.0, f"Nk {Nk} n_ip {n_ip} ip_scale {ip_scale}: err / bar {r:.3f}"
            worst = max(worst, r)
            if ip_scale == 0.0 and n_ip:
                v2 = v.clone().view(B, Nk, -1)
                v2[:, Nk - n_ip:] *= 2
                out2 = ops.attention(q, k, v2.view(B * Nk, -1), B, H, Nq, Nk, n_ip=n_ip, ip_scale=0.0)
                assert torch.equal(out, out2), f"Nk {Nk} n_ip {n_ip}: the image-prompt part leaks at ip_scale 0"
    report(f"attention two-segment {Nq}x{Nk}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# guidance-rescale statistics of the step kernels
# ---------------------------------------------------------------------------------------------------------------------
def _check(out, ref, what):
    """test_kernels_gpu.check at the bar every rescale step test uses (rtol = atol = 2e-3)."""
    close_ulps(out, ref, what, ulps=0.0, slack=2e-3 + (2e-3 + 2.0 ** -11) * ref.double().abs())


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("hw", STEP_BUCKETS)
def test_step_kernels_rescale_planted(ops, n, hw):
    """ih_euler_step_ex, ih_euler_inpaint_step, ih_dpm_solver_step and ih_euler_ancestral_step with guidance_rescale
    0.7 on planted noise predictions (latents 0), against each kernel test's own fp16 rounding-point reference."""
    from dpm_ref import dpm_step_ref
    from euler_a_ref import euler_a_step_ref
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from inpaint_ref import inpaint_step_ref
    from oracle.scheduler_ref import rescale_noise_cfg
    h, w = hw
    T, i, r = 10, 4, 0.7
    noise = P.rescale_build(n, h, w, device="cuda")
    zeros = torch.zeros(n, 4, h, w, dtype=torch.float16, device="cuda")
    tag = f"n{n} {h}x{w}"
    # Euler (test_kernels_gpu.py::test_euler_step_ex)
    sig = torch.tensor([13.1204, 11.6761, 10.4250, 0.0], device="cuda")
    lat, mi = zeros.clone(), torch.empty(2 * n, 4, h, w, dtype=torch.float16, device="cuda")
    ops.euler_step(noise, lat, mi, sig, torch.tensor([1], dtype=torch.int32, device="cuda"), 5.0,
                   guidance_rescale=r)
    u, c = noise.chunk(2)
    eps = rescale_noise_cfg(u + 5.0 * (c - u), c, r)
    x0 = -(sig[1] * eps.float()).half().float()
    _check(lat, (-x0 / sig[1] * (sig[2] - sig[1])).half(), f"euler_step_ex {tag}")
    # inpainting Euler, mask 1 (test_inpaint_gpu.py::test_euler_inpaint_step_kernel)
    sig_np = EulerDiscreteScheduler().set_timesteps(T).sigmas
    ones = torch.ones(n, 1, h, w, dtype=torch.float16, device="cuda")
    ref_x, _ = inpaint_step_ref(noise, zeros, sig_np, i, 7.5, zeros, zeros, ones, T, True, r)
    lat = zeros.clone()
    ops.euler_inpaint_step(noise, lat, mi, torch.from_numpy(sig_np).cuda(),
                           torch.tensor([i], dtype=torch.int32, device="cuda"), 7.5, zeros, zeros, ones,
                           torch.tensor([T], dtype=torch.int32, device="cuda"), guidance_rescale=r)
    _check(lat, ref_x, f"euler_inpaint_step {tag}")
    # DPM-Solver++ 2M, second order (test_dpm_gpu.py::test_dpm_solver_step_kernel)
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(T)
    prev = P.rescale_build(n, h, w, device="cuda")[n:]
    ref_x, ref_x0, _ = dpm_step_ref(noise, zeros, prev, T, False, i, False, 7.5, True, r)
    lat, x0 = zeros.clone(), prev.clone()
    ops.dpm_solver_step(noise, lat, mi, x0, torch.from_numpy(s.coeffs).cuda(),
                        torch.tensor([i], dtype=torch.int32, device="cuda"),
                        torch.tensor([0], dtype=torch.int32, device="cuda"), 7.5, guidance_rescale=r)
    _check(x0, ref_x0, f"dpm_solver_step x0 {tag}")
    _check(lat, ref_x, f"dpm_solver_step {tag}")
    # Euler Ancestral, step noise 0 (test_euler_a_gpu.py::test_euler_ancestral_step_kernel)
    sa = EulerAncestralDiscreteScheduler()
    sa.set_timesteps(T)
    step_noise = torch.zeros(T, n, 4, h, w, dtype=torch.float16, device="cuda")
    ref_x, _ = euler_a_step_ref(noise, zeros, T, i, 7.5, step_noise[i], True, r)
    lat = zeros.clone()
    ops.euler_ancestral_step(noise, lat, mi, torch.from_numpy(sa.coeffs).cuda(), step_noise,
                             torch.tensor([i], dtype=torch.int32, device="cuda"), 7.5, guidance_rescale=r)
    _check(lat, ref_x, f"euler_ancestral_step {tag}")
