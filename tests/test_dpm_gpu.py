"""GPU tests of DPM-Solver++ 2M: the step kernel against the torch restatement of diffusers' step on the same fp16
tensors and 0-dim scalars (tests/dpm_ref.py), TINY trajectories (graph and eager) against the fp32 oracle, graph reuse
across scheduler swaps and batch sizes, SDXL-base trajectories, and IPAdapterXL.generate over a DPM pipeline."""
import pytest
import torch

from test_kernels_gpu import STEP_BUCKETS, check, ops  # noqa: F401  (fixture)
from test_unet_gpu import _errs, _inputs, _make_pair, sdxl_pair  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("use_cfg,rescale,hw", [
    pytest.param(True, 0.0, (64, 48), id="True-0.0"), pytest.param(False, 0.0, (64, 48), id="False-0.0"),
    pytest.param(True, 0.7, (64, 48), id="True-0.7"),
] + [pytest.param(True, 0.7, hw, id=f"True-0.7-{hw[0]}x{hw[1]}") for hw in STEP_BUCKETS])
def test_dpm_solver_step_kernel(ops, use_cfg, rescale, n, karras, hw):  # noqa: F811
    """First order at loop_begin (index 0, and mid-schedule with loop_begin there), second order mid-schedule, and the
    final step to sigma 0, which must return x0 exactly.  Without rescale bit-exact against diffusers' expressions
    on the same fp16 CUDA tensors and 0-dim CPU scalars; with rescale the bar of test_kernels_gpu.py::test_euler_step_ex
    (the per-image std is a reduction in another order than torch's)."""
    from dpm_ref import dpm_step_ref
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    T, (h, w) = 10, hw
    s = DPMSolverMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    coeffs = torch.from_numpy(s.coeffs).cuda()
    b = 2 * n if use_cfg else n
    g = torch.Generator().manual_seed(100 * n + 10 * int(use_cfg) + int(karras))
    for i, begin in ((0, 0), (4, 0), (4, 4), (8, 0), (9, 0)):
        sig = float(s.sigmas[i])
        lat = (torch.randn(n, 4, h, w, generator=g) * min(sig, 1.0)).half().cuda()
        noise_pred = torch.randn(b, 4, h, w, generator=g).half().cuda()
        prev = torch.randn(n, 4, h, w, generator=g).half().cuda()
        first = i == begin
        ref_x, ref_x0, ref_mi = dpm_step_ref(noise_pred, lat, prev, T, karras, i, first, 7.5, use_cfg, rescale)
        step = torch.tensor([i], dtype=torch.int32, device="cuda")
        loop_begin = torch.tensor([begin], dtype=torch.int32, device="cuda")
        model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
        x0 = prev.clone()
        ops.dpm_solver_step(noise_pred, lat, model_in, x0, coeffs, step, loop_begin, 7.5, use_cfg=use_cfg,
                            guidance_rescale=rescale)
        assert int(step.item()) == i + 1 and int(loop_begin.item()) == begin
        what = f"dpm cfg={use_cfg} r={rescale} n={n} karras={karras} step {i} begin {begin}"
        if rescale == 0.0:
            exact = (lat == ref_x).float().mean().item()
            print(f"[{what}] bit-exact latents {exact:.6f}")
            assert torch.equal(x0, ref_x0), what + " x0"
            assert torch.equal(lat, ref_x) and torch.equal(model_in, ref_mi), what
        else:
            check(x0, ref_x0, what + " x0", rtol=2e-3, atol=2e-3)
            check(lat, ref_x, what, rtol=2e-3, atol=2e-3)
            check(model_in, ref_mi, what + " model_in", rtol=2e-3, atol=2e-3)
        if i == T - 1:
            assert torch.equal(lat, x0), "the step to sigma 0 returns x0"


def _tiny_oracle_run(m, dev, dt, latents, pos, neg, ppool, npool, tid, T, karras, **kw):
    from dpm_ref import dpm_denoise_loop
    procs = [p for p in m.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    fn = lambda s, t, e, te, ti: m(s.to(dt), t, e, te, ti).to(torch.float16)  # noqa: E731
    return dpm_denoise_loop(fn, latents.to(dev), pos.to(dev, dt), neg.to(dev, dt), ppool.to(dev, dt), npool.to(dev, dt),
                            tid.to(dev), T, karras=karras, set_scale=set_scale, **kw)


@pytest.mark.parametrize("karras", [False, True])
def test_dpm_tiny_trajectory_matches_oracle(karras):
    """DPM++ 2M at T = 6, CFG 5.0, IP scale 0.8 gated off at the end, denoising_end 0.8: native eager and graph-replayed
    vs the fp32 CPU oracle with the bar of SURVEY section 7; the graph replay is bit-identical to the eager run and to a
    second replay."""
    from dpm_ref import DPMSolverRef, denoising_end_steps
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    native, ref32, eager16 = _make_pair(TINY, seed=31)
    T, n, lat = 6, 2, 32
    latents = prepare_latents(n, 4, lat, lat, [42, 43], 1.0)
    x = _inputs(TINY, n, lat, seed=33)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    kw = dict(guidance_scale=5.0, conditioning_scale=0.8, control_guidance_end=0.7, denoising_end=0.8)
    r = _tiny_oracle_run(ref32, "cpu", torch.float32, latents, *args, T, karras, **kw)
    e = _tiny_oracle_run(eager16, "cuda", torch.float16, latents, *args, T, karras, **kw)
    loop_steps = denoising_end_steps(DPMSolverRef(T, karras).timesteps.tolist(), 0.8)
    assert 1 < loop_steps < T
    outs = []
    for use_graph in (False, True, True):
        eng = DenoiseEngine(native, use_cuda_graph=use_graph, scheduler=DPMSolverMultistepScheduler(use_karras_sigmas=karras))
        calls = []
        o = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, control_guidance_end=0.7,
                    num_loop_steps=loop_steps, callback=lambda i, t, lt: calls.append(i))
        torch.cuda.synchronize()
        assert calls == list(range(loop_steps))
        e_nat, e_eag, mx = _errs(o, r, e)
        print(f"[dpm tiny karras={karras} graph={use_graph}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  "
              f"max|ref| {mx:.3e}")
        assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
        outs.append(o)
        if use_graph:
            o2 = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, control_guidance_end=0.7,
                         num_loop_steps=loop_steps)
            assert torch.equal(o, o2), "a second replay must reproduce the first"
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), "graph replay must equal the eager run"


def test_scheduler_swaps_and_batch_changes_bit_equal_to_fresh_pipelines():
    """Euler -> DPM (Karras) -> Euler on one pipeline, and n = 1 -> 3 -> 1 with DPM: each call bit-identical to the
    same call on a fresh pipeline over the same UNet."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
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

    def karras():
        return DPMSolverMultistepScheduler.from_config(EulerDiscreteScheduler().config, use_karras_sigmas=True)
    pipe = StableDiffusionXLCustomPipeline(native)
    got = [call(pipe, 1)]
    pipe.scheduler = karras()
    got.append(call(pipe, 1))
    got += [call(pipe, 3), call(pipe, 1)]
    pipe.scheduler = EulerDiscreteScheduler()
    got.append(call(pipe, 1))
    torch.cuda.synchronize()
    fresh = [call(StableDiffusionXLCustomPipeline(native), 1), call(StableDiffusionXLCustomPipeline(native, scheduler=karras()), 1),
             call(StableDiffusionXLCustomPipeline(native, scheduler=karras()), 3)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], fresh[0]) and torch.equal(got[4], fresh[0])
    assert torch.equal(got[1], fresh[1]) and torch.equal(got[3], fresh[1])
    assert torch.equal(got[2], fresh[2])
    assert not torch.equal(got[0], got[1])


def test_dpm_karras_sdxl_base_512_matches_oracle(sdxl_pair):  # noqa: F811
    """SDXL-base at 512^2: a 4-step DPM++ 2M Karras trajectory (CFG 5.0) through the CUDA-graph loop vs the CPU fp32
    oracle, bar of SURVEY section 7; then a graph-replayed 1024^2 20-step run comes out finite."""
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    cfg, native, ref, eager16 = sdxl_pair
    T, n, lat = 4, 1, 64
    latents = prepare_latents(n, 4, lat, lat, [42], 1.0)
    x = _inputs(cfg, n, lat, seed=13)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    with torch.no_grad():
        r4 = _tiny_oracle_run(ref, "cpu", torch.float32, latents, *args, T, True, guidance_scale=5.0)
        e4 = _tiny_oracle_run(eager16, "cuda", torch.float16, latents, *args, T, True, guidance_scale=5.0)
    eng = DenoiseEngine(native, scheduler=DPMSolverMultistepScheduler(use_karras_sigmas=True))
    o4 = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=1.0)
    torch.cuda.synchronize()
    e_nat, e_eag, mx = _errs(o4, r4, e4)
    print(f"[DPM++ 2M Karras SDXL-base 512^2, 4 steps] native max|err| {e_nat:.3e}  eager-fp16 {e_eag:.3e}  "
          f"max|ref| {mx:.3e}")
    assert torch.isfinite(o4).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)

    lat = 128
    big = prepare_latents(n, 4, lat, lat, [7], 1.0)
    xb = _inputs(cfg, n, lat, seed=17)
    o = eng.run(big.pin_memory(), xb["ehs"][n:], xb["ehs"][:n], xb["text_embeds"][n:], xb["text_embeds"][:n],
                xb["time_ids"][:n], 20, guidance_scale=5.0, ip_scale=1.0)
    torch.cuda.synchronize()
    print(f"[DPM++ 2M Karras SDXL-base 1024^2, 20 steps] max|latent| {o.float().abs().max().item():.3e}")
    assert torch.isfinite(o).all()


def test_ip_adapter_xl_generate_dpm_tiny_matches_oracle():
    """IPAdapterXL.generate over a TINY pipeline with DPM++ 2M Karras: the oracle pipeline from oracle/ parts with the
    same weights and the dpm_ref loop."""
    from dpm_ref import dpm_denoise_loop
    from imagharmony_b200.config import HARMONY_TINY, TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    from train import HarmonyAttention

    cfg, h = TINY, HARMONY_TINY
    with torch.device("meta"):
        shapes = shapes_of(UNetRef(cfg))
    sd = random_state_dict(shapes, 11)
    pipe = StableDiffusionXLCustomPipeline(UNet2DConditionModel.from_state_dict(cfg, sd, device="cuda"))
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config, use_karras_sigmas=True)
    kw = dict(image_hidden_size=h.image_hidden_size, text_context_dim=h.text_context_dim, inter_dim=h.inter_dim,
              cross_heads=h.cross_heads, reshape_blocks=h.reshape_blocks, cross_value_dim=h.cross_value_dim, scale=1.0)
    ha = HarmonyAttention(fusion_method="cross_attention", **kw)
    ip_model = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4, inference=True, number_class_crossattention=ha)
    ck = {"image_proj": random_state_dict(shapes_of(ip_model.image_proj_model), 3),
          "composed_adapter": random_state_dict(shapes_of(ha), 4),
          "ip_adapter": random_state_dict(shapes_of(torch.nn.ModuleList(pipe.unet.attn_processors.values())), 5)}
    ip_model.image_proj_model.load_state_dict({k: v.cuda() for k, v in ck["image_proj"].items()})
    ip_model.number_class_crossattention.load_state_dict({k: v.cuda() for k, v in ck["composed_adapter"].items()})
    torch.nn.ModuleList(pipe.unet.attn_processors.values()).load_state_dict({k: v.cuda() for k, v in ck["ip_adapter"].items()})
    pipe.unet.finalize()
    img = torch.randn(1, h.image_hidden_size, generator=torch.Generator("cpu").manual_seed(5)).half()
    T, res = 4, 256
    out = ip_model.generate(pil_image=None, clip_image_embeds=img, prompt="lions", negative_prompt="blurry", scale=0.8,
                            guidance_scale=5.0, num_samples=1, num_inference_steps=T, seed=[42], extra_text="eight sheep",
                            output_type="latent", height=res, width=res)
    torch.cuda.synchronize()
    ref_unet = UNetRef(cfg)
    ref_unet.load_state_dict({k: v.float() for k, v in sd.items()})
    pr = A.install_processors(ref_unet, cfg)
    torch.nn.ModuleList(pr.values()).load_state_dict({k: v.float() for k, v in ck["ip_adapter"].items()})
    ref_unet.eval()
    rha = A.HarmonyAttentionRef(**kw)
    rha.load_state_dict({k: v.float() for k, v in ck["composed_adapter"].items()})
    rip = A.ImageProjRef(cfg.cross_attention_dim, h.image_hidden_size, 4)
    rip.load_state_dict({k: v.float() for k, v in ck["image_proj"].items()})
    enc = pipe.prompt_encoder
    pe, pp = enc(["lions"])
    ne, npool = enc(["blurry"])
    xe, _ = enc(["eight sheep"])
    with torch.no_grad():
        emb = img.float() + rha(xe.float(), img.float())
        cond, uncond = rip(emb), rip(torch.zeros_like(emb))
    pos = torch.cat([pe.float(), cond], dim=1)
    neg = torch.cat([ne.float(), uncond], dim=1)
    lat = torch.randn((1, 4, res // 8, res // 8), generator=torch.Generator("cpu").manual_seed(42)).half()
    tid = torch.tensor([[res, res, 0, 0, res, res]], dtype=torch.float32)
    for p in (p for p in ref_unet.attn_processors.values() if hasattr(p, "to_k_ip")):
        p.scale = 0.8
    want = dpm_denoise_loop(lambda s, t, e, a, b: ref_unet(s.float(), t, e, a, b).half(), lat, pos, neg, pp.float(),
                            npool.float(), tid, T, karras=True, guidance_scale=5.0)
    err = (out.float().cpu() - want.float()).abs().max().item()
    mx = want.float().abs().max().item()
    print(f"[IPAdapterXL.generate DPM tiny] max|err| {err:.3e} max|ref| {mx:.3e}")
    assert err <= 2e-2 * mx, (err, mx)
