"""GPU tests of Euler Ancestral: the step kernel against diffusers' step run by torch on the same fp16 CUDA tensors,
0-dim CPU scalars and noise (tests/euler_a_ref.py), TINY trajectories (graph and eager; text-to-image, image-to-image,
inpainting) against the fp32 oracle with the same noise, graph reuse across scheduler swaps, batch sizes and a stop /
resume, an SDXL-base trajectory, and IPAdapterXL.generate over an Euler A pipeline."""
import pytest
import torch

from test_kernels_gpu import STEP_BUCKETS, check, ops  # noqa: F401  (fixture)
from test_unet_gpu import _errs, _inputs, _make_pair, sdxl_pair  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _table(T):
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    s = EulerAncestralDiscreteScheduler()
    s.set_timesteps(T)
    return s, torch.from_numpy(s.coeffs).cuda()


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("use_cfg,rescale,hw", [
    pytest.param(True, 0.0, (64, 48), id="True-0.0"), pytest.param(False, 0.0, (64, 48), id="False-0.0"),
    pytest.param(True, 0.7, (64, 48), id="True-0.7"),
] + [pytest.param(True, 0.7, hw, id=f"True-0.7-{hw[0]}x{hw[1]}") for hw in STEP_BUCKETS])
def test_euler_ancestral_step_kernel(ops, use_cfg, rescale, n, hw):  # noqa: F811
    """First, middle and last index.  Without rescale bit-exact against diffusers' expressions on the same fp16 CUDA
    tensors, 0-dim CPU scalars and noise; with rescale the bar of test_kernels_gpu.py::test_euler_step_ex."""
    from euler_a_ref import euler_a_step_ref
    T, (h, w) = 10, hw
    s, coeffs = _table(T)
    b = 2 * n if use_cfg else n
    g = torch.Generator().manual_seed(100 * n + 10 * int(use_cfg) + int(rescale > 0))
    step_noise = torch.randn(T, n, 4, h, w, generator=g).half().cuda()
    for i in (0, 4, T - 1):
        lat = (torch.randn(n, 4, h, w, generator=g) * float(s.sigmas[i])).half().cuda()
        noise_pred = torch.randn(b, 4, h, w, generator=g).half().cuda()
        ref_x, ref_mi = euler_a_step_ref(noise_pred, lat, T, i, 7.5, step_noise[i], use_cfg, rescale)
        step = torch.tensor([i], dtype=torch.int32, device="cuda")
        model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
        ops.euler_ancestral_step(noise_pred, lat, model_in, coeffs, step_noise, step, 7.5, use_cfg=use_cfg,
                                 guidance_rescale=rescale)
        assert int(step.item()) == i + 1
        what = f"euler_a cfg={use_cfg} r={rescale} n={n} step {i}"
        if rescale == 0.0:
            print(f"[{what}] bit-exact latents {(lat == ref_x).float().mean().item():.6f}")
            assert torch.equal(lat, ref_x) and torch.equal(model_in, ref_mi), what
        else:
            check(lat, ref_x, what, rtol=2e-3, atol=2e-3)
            check(model_in, ref_mi, what + " model_in", rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("use_cfg", [True, False])
@pytest.mark.parametrize("binary", [True, False])
def test_euler_ancestral_step_kernel_with_blend(ops, binary, use_cfg):  # noqa: F811
    """The inpainting blend after the ancestral step, bit-exact: re-noised image latents mid-loop, the clean ones at
    blend_end - 1 (denoising_end) and at the end of the schedule; binary and fractional masks."""
    from euler_a_ref import euler_a_step_ref
    T, n, h, w = 10, 2, 32, 40
    s, coeffs = _table(T)
    b = 2 * n if use_cfg else n
    g = torch.Generator().manual_seed(7 + int(binary) + 2 * int(use_cfg))
    step_noise = torch.randn(T, n, 4, h, w, generator=g).half().cuda()
    img = torch.randn(n, 4, h, w, generator=g).half().cuda()
    bnoise = torch.randn(n, 4, h, w, generator=g).half().cuda()
    m = torch.rand(n, 1, h, w, generator=g)
    mask = ((m > 0.5).float() if binary else m).half().cuda()
    for i, end in ((3, 10), (5, 6), (9, 10)):
        lat = (torch.randn(n, 4, h, w, generator=g) * float(s.sigmas[i])).half().cuda()
        noise_pred = torch.randn(b, 4, h, w, generator=g).half().cuda()
        ref_x, ref_mi = euler_a_step_ref(noise_pred, lat, T, i, 5.0, step_noise[i], use_cfg,
                                         blend=(img, bnoise, mask), blend_end=end)
        step = torch.tensor([i], dtype=torch.int32, device="cuda")
        blend_end = torch.tensor([end], dtype=torch.int32, device="cuda")
        model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
        ops.euler_ancestral_step(noise_pred, lat, model_in, coeffs, step_noise, step, 5.0, use_cfg=use_cfg,
                                 inpaint=(img, bnoise, mask, blend_end))
        what = f"euler_a blend binary={binary} cfg={use_cfg} step {i} end {end}"
        assert torch.equal(lat, ref_x) and torch.equal(model_in, ref_mi), what


@pytest.mark.parametrize("i", [0, 3, 9])
def test_first_input_equals_torch_scale_model_input(ops, i):  # noqa: F811
    """The loop's first model input equals diffusers' scale_model_input as torch evaluates it on the same tensor."""
    from euler_a_ref import EulerAncestralRef
    T = 10
    _, coeffs = _table(T)
    lat = (torch.randn(3, 4, 64, 48, generator=torch.Generator().manual_seed(i)) * 8).half().cuda()
    sched = EulerAncestralRef(T)
    sched.step_index = i
    want = sched.scale_model_input(lat)
    model_in = torch.empty(6, 4, 64, 48, dtype=torch.float16, device="cuda")
    ops.euler_ancestral_scale_input(lat, model_in, coeffs, torch.tensor([i], dtype=torch.int32, device="cuda"))
    assert torch.equal(model_in, torch.cat([want, want]))


def _oracle(m, dev, dt, latents, pos, neg, ppool, npool, tid, T, seed, **kw):
    from euler_a_ref import euler_a_denoise_loop
    procs = [p for p in m.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    fn = lambda s, t, e, te, ti: m(s.to(dt), t, e, te, ti).to(torch.float16)  # noqa: E731
    return euler_a_denoise_loop(fn, latents.to(dev), pos.to(dev, dt), neg.to(dev, dt), ppool.to(dev, dt),
                                npool.to(dev, dt), tid.to(dev), T, generator=torch.Generator().manual_seed(seed),
                                set_scale=set_scale, **kw)


def _tiny(seed=31, n=2, lat=32):
    from imagharmony_b200.config import TINY
    native, ref32, eager16 = _make_pair(TINY, seed=seed)
    x = _inputs(TINY, n, lat, seed=33)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    return native, ref32, eager16, args


def test_euler_a_tiny_trajectory_matches_oracle():
    """T = 6, CFG 5.0, IP scale 0.8 gated off at the end, denoising_end 0.8, a CPU generator: native eager and
    graph-replayed vs the fp32 oracle drawing the same noise, bar of SURVEY section 7; the graph replay equals the
    eager run and a second replay bit for bit; another seed gives another result."""
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from oracle.scheduler_ref import denoising_end_steps, euler_tables, prepare_latents
    native, ref32, eager16, args = _tiny()
    T, n = 6, 2
    latents = prepare_latents(n, 4, 32, 32, [42, 43], euler_tables(T)[2])
    kw = dict(guidance_scale=5.0, conditioning_scale=0.8, control_guidance_end=0.7, denoising_end=0.8)
    r = _oracle(ref32, "cpu", torch.float32, latents, *args, T, 5, **kw)
    e = _oracle(eager16, "cuda", torch.float16, latents, *args, T, 5, **kw)
    loop_steps = denoising_end_steps(T, 0.8)
    assert 1 < loop_steps < T
    outs = []

    def run(eng, seed, **extra):
        return eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, control_guidance_end=0.7,
                       num_loop_steps=loop_steps, generator=torch.Generator().manual_seed(seed), **extra)
    for use_graph in (False, True, True):
        eng = DenoiseEngine(native, use_cuda_graph=use_graph, scheduler=EulerAncestralDiscreteScheduler())
        calls = []
        o = run(eng, 5, callback=lambda i, t, lt: calls.append(i))
        torch.cuda.synchronize()
        assert calls == list(range(loop_steps))
        e_nat, e_eag, mx = _errs(o, r, e)
        print(f"[euler_a tiny graph={use_graph}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  max|ref| {mx:.3e}")
        assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
        outs.append(o)
        if use_graph:
            assert torch.equal(o, run(eng, 5)), "a second replay must reproduce the first"
            assert (run(eng, 6).float() - o.float()).abs().max() > 1e-2, "another seed must change the result"
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), "graph replay must equal the eager run"


def test_euler_a_tiny_img2img_and_inpaint_match_oracle():
    """Graph-replayed image-to-image (begin_step) and inpainting (blend) vs the oracle with the same noise; an all-one
    mask reproduces image-to-image bit for bit, an all-zero mask returns the clean image latents."""
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    native, ref32, eager16, args = _tiny(seed=37)
    T, n, begin = 6, 2, 2
    g = torch.Generator().manual_seed(9)
    img = (torch.randn(n, 4, 32, 32, generator=g) * 0.8).half()
    bnoise = torch.randn(n, 4, 32, 32, generator=g).half()
    mask = (torch.rand(n, 1, 32, 32, generator=g) > 0.4).half()
    from euler_a_ref import EulerAncestralRef
    from img2img_ref import add_noise_ref
    start = add_noise_ref(img, bnoise, float(EulerAncestralRef(T).sigmas[begin]))
    eng = DenoiseEngine(native, scheduler=EulerAncestralDiscreteScheduler())

    def run(inpaint=None):
        return eng.run(start.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, begin_step=begin,
                       inpaint=inpaint, generator=torch.Generator().manual_seed(3))
    for blend in (None, (img, bnoise, mask)):
        kw = dict(guidance_scale=5.0, conditioning_scale=0.8, begin=begin)
        kw32 = dict(kw, blend=None if blend is None else tuple(t.float() for t in blend))
        kw16 = dict(kw, blend=None if blend is None else tuple(t.cuda() for t in blend))
        r = _oracle(ref32, "cpu", torch.float32, start, *args, T, 3, **kw32)
        e = _oracle(eager16, "cuda", torch.float16, start, *args, T, 3, **kw16)
        o = run(None if blend is None else tuple(t.cuda() for t in blend))
        torch.cuda.synchronize()
        e_nat, e_eag, mx = _errs(o, r, e)
        print(f"[euler_a tiny {'inpaint' if blend else 'img2img'}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  "
              f"max|ref| {mx:.3e}")
        assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
    i2i = run()
    ones = run((img.cuda(), bnoise.cuda(), torch.ones_like(mask).cuda()))
    zeros = run((img.cuda(), bnoise.cuda(), torch.zeros_like(mask).cuda()))
    torch.cuda.synchronize()
    assert torch.equal(ones, i2i) and torch.equal(zeros, img.cuda())


def test_scheduler_swaps_batch_changes_and_resume_bit_equal_to_fresh_runs():
    """Euler -> Euler A -> DPM -> Euler on one pipeline, and n = 1 -> 3 -> 1 with Euler A: each call bit-identical to
    the same call on a fresh pipeline; a graph-replayed stop_after / start_step pair on one continuing generator equals
    the uninterrupted run."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    native, _, _ = _make_pair(TINY, seed=35)
    g = torch.Generator().manual_seed(11)
    emb = {k: torch.randn(3, *s, generator=g).half() for k, s in (
        ("prompt_embeds", (81, TINY.cross_attention_dim)), ("negative_prompt_embeds", (81, TINY.cross_attention_dim)),
        ("pooled_prompt_embeds", (TINY.pooled_embed_dim,)), ("negative_pooled_prompt_embeds", (TINY.pooled_embed_dim,)))}

    def call(pipe, n):
        pipe.set_scale(0.7)
        return pipe(num_inference_steps=5, height=128, width=128, guidance_scale=5.0, control_guidance_end=0.7,
                    generator=[torch.Generator().manual_seed(s) for s in range(n)], output_type="latent",
                    **{k: v[:n] for k, v in emb.items()}).images

    def anc():
        return EulerAncestralDiscreteScheduler.from_config(EulerDiscreteScheduler().config)
    pipe = StableDiffusionXLCustomPipeline(native)
    got = [call(pipe, 1)]
    pipe.scheduler = anc()
    got += [call(pipe, 1), call(pipe, 3), call(pipe, 1)]
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)
    got.append(call(pipe, 1))
    pipe.scheduler = EulerDiscreteScheduler()
    got.append(call(pipe, 1))
    torch.cuda.synchronize()
    fresh = [call(StableDiffusionXLCustomPipeline(native), 1), call(StableDiffusionXLCustomPipeline(native, scheduler=anc()), 1),
             call(StableDiffusionXLCustomPipeline(native, scheduler=anc()), 3),
             call(StableDiffusionXLCustomPipeline(native, scheduler=DPMSolverMultistepScheduler()), 1)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], fresh[0]) and torch.equal(got[5], fresh[0])
    assert torch.equal(got[1], fresh[1]) and torch.equal(got[3], fresh[1])
    assert torch.equal(got[2], fresh[2]) and torch.equal(got[4], fresh[3])
    assert not torch.equal(got[0], got[1])

    x = _inputs(TINY, 2, 16, seed=5)
    args = (x["ehs"][2:], x["ehs"][:2], x["text_embeds"][2:], x["text_embeds"][:2], x["time_ids"][:2], 6)
    lat = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(1)).half() * 9
    eng = DenoiseEngine(native, scheduler=anc())
    full = eng.run(lat, *args, generator=torch.Generator().manual_seed(4))
    gen = torch.Generator().manual_seed(4)
    part = eng.run(lat, *args, stop_after=3, generator=gen)
    rest = eng.run(part, *args, start_step=3, generator=gen)
    torch.cuda.synchronize()
    assert torch.equal(rest, full)


def test_euler_a_sdxl_base_512_matches_oracle(sdxl_pair):  # noqa: F811
    """SDXL-base at 512^2: a 4-step Euler A trajectory (CFG 5.0, seeded CPU generator) through the CUDA-graph loop vs
    the CPU fp32 oracle drawing the same noise, bar of SURVEY section 7."""
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from oracle.scheduler_ref import euler_tables, prepare_latents
    cfg, native, ref, eager16 = sdxl_pair
    T, n, lat = 4, 1, 64
    latents = prepare_latents(n, 4, lat, lat, [42], euler_tables(T)[2])
    x = _inputs(cfg, n, lat, seed=13)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    with torch.no_grad():
        r4 = _oracle(ref, "cpu", torch.float32, latents, *args, T, 8, guidance_scale=5.0)
        e4 = _oracle(eager16, "cuda", torch.float16, latents, *args, T, 8, guidance_scale=5.0)
    eng = DenoiseEngine(native, scheduler=EulerAncestralDiscreteScheduler())
    o4 = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=1.0,
                 generator=torch.Generator().manual_seed(8))
    torch.cuda.synchronize()
    e_nat, e_eag, mx = _errs(o4, r4, e4)
    print(f"[Euler A SDXL-base 512^2, 4 steps] native max|err| {e_nat:.3e}  eager-fp16 {e_eag:.3e}  max|ref| {mx:.3e}")
    assert torch.isfinite(o4).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)


def test_ip_adapter_xl_generate_euler_a_tiny():
    """IPAdapterXL.generate over a TINY Euler A pipeline: seeded, finite, repeatable, and not Euler's result."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    native, _, _ = _make_pair(TINY, seed=41)
    pipe = StableDiffusionXLCustomPipeline(native)
    ip_model = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0)).half()
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=42,
                  output_type="latent", height=128, width=128)
    euler = ip_model.generate(**common)
    pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    a, b = ip_model.generate(**common), ip_model.generate(**common)
    torch.cuda.synchronize()
    assert a.shape == (2, 4, 16, 16) and torch.isfinite(a.float()).all() and torch.equal(a, b)
    assert (a.float() - euler.float()).abs().max() > 1e-2
