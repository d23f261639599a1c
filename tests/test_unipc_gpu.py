"""GPU tests of UniPC: the step kernel against the torch restatement of diffusers' step on the same fp16 tensors and
0-dim scalars (tests/unipc_ref.py), stale history that a step must not read, TINY trajectories (graph and eager)
against the fp32 oracle, graph reuse across scheduler swaps and batch sizes, an SDXL-base trajectory, a ControlNet
loop, and IPAdapterXL.generate over a UniPC pipeline."""
import pytest
import torch

from test_kernels_gpu import STEP_BUCKETS, check, ops  # noqa: F401  (fixture)
from test_unet_gpu import _errs, _inputs, _make_pair, sdxl_pair  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

T_KERNEL = 10


def _step_case(s, i, n, b, h, w, g):
    """Latents at sigma_i's scale, a noise prediction and a history of plausible magnitude."""
    sig = float(s.sigmas[i])
    lat = (torch.randn(n, 4, h, w, generator=g) * max(min(sig, 1.0), 0.3)).half().cuda()
    noise_pred = torch.randn(b, 4, h, w, generator=g).half().cuda()
    last = (torch.randn(n, 4, h, w, generator=g) * max(min(sig, 1.0), 0.3)).half().cuda()
    x0_1 = torch.randn(n, 4, h, w, generator=g).half().cuda()
    x0_2 = torch.randn(n, 4, h, w, generator=g).half().cuda()
    return lat, noise_pred, last, x0_1, x0_2


def _run_kernel(ops, s, coeffs, i, begin, lat, noise_pred, last, x0_1, x0_2, use_cfg, rescale):  # noqa: F811
    b = noise_pred.shape[0]
    n, _, h, w = lat.shape
    step = torch.tensor([i], dtype=torch.int32, device="cuda")
    loop_begin = torch.tensor([begin], dtype=torch.int32, device="cuda")
    model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
    out = {"latents": lat.clone(), "last_sample": last.clone(), "prev_x0": x0_1.clone(), "prev_x0_2": x0_2.clone()}
    ops.dpm_solver_step(noise_pred, out["latents"], model_in, out["prev_x0"], coeffs, step, loop_begin, 7.5,
                        use_cfg=use_cfg, guidance_rescale=rescale, unipc=(out["last_sample"], out["prev_x0_2"]))
    assert int(step.item()) == i + 1 and int(loop_begin.item()) == begin
    out["model_in"] = model_in
    return out


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("use_cfg,rescale,hw", [
    pytest.param(True, 0.0, (64, 48), id="True-0.0"), pytest.param(False, 0.0, (64, 48), id="False-0.0"),
    pytest.param(True, 0.7, (64, 48), id="True-0.7"),
] + [pytest.param(True, 0.0, hw, id=f"True-0.0-{hw[0]}x{hw[1]}") for hw in STEP_BUCKETS]
  + [pytest.param(True, 0.7, hw, id=f"True-0.7-{hw[0]}x{hw[1]}") for hw in STEP_BUCKETS])
def test_unipc_step_kernel(ops, use_cfg, rescale, n, karras, hw):  # noqa: F811
    """Steps 0, 1, 2, mid, T-2, T-1 of a loop from index 0, and the first two steps of a loop begun mid-schedule.
    Without rescale every output (latents, last_sample, prev_x0, prev_x0_2, model_in) is bit-exact against diffusers'
    expressions on the same fp16 CUDA tensors and 0-dim CPU scalars; with rescale the bar of test_dpm_solver_step_kernel
    applies.  The step to sigma 0 returns x0 exactly."""
    from unipc_ref import unipc_step_ref
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    T, (h, w) = T_KERNEL, hw
    s = UniPCMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    coeffs = torch.from_numpy(s.coeffs).cuda()
    b = 2 * n if use_cfg else n
    g = torch.Generator().manual_seed(100 * n + 10 * int(use_cfg) + int(karras))
    for i, begin in ((0, 0), (1, 0), (2, 0), (5, 0), (T - 2, 0), (T - 1, 0), (5, 5), (6, 5)):
        case = _step_case(s, i, n, b, h, w, g)
        lat, noise_pred, last, x0_1, x0_2 = case
        want = dict(zip(("latents", "last_sample", "prev_x0", "prev_x0_2", "model_in"),
                        unipc_step_ref(noise_pred, lat, last, x0_1, x0_2, T, karras, i, begin, 7.5, use_cfg, rescale)))
        got = _run_kernel(ops, s, coeffs, i, begin, *case, use_cfg, rescale)
        what = f"unipc cfg={use_cfg} r={rescale} n={n} karras={karras} {h}x{w} step {i} begin {begin}"
        assert torch.equal(got["prev_x0_2"], x0_1), what + " prev_x0_2 <- prev_x0"
        for k in want:
            if rescale == 0.0:
                assert torch.equal(got[k], want[k]), f"{what} {k}"
            else:
                check(got[k], want[k], f"{what} {k}", rtol=2e-3, atol=2e-3)
        if i == T - 1:
            assert torch.equal(got["latents"], got["prev_x0"]), "the step to sigma 0 returns x0"


@pytest.mark.parametrize("use_cfg,rescale", [(True, 0.0), (True, 0.7), (False, 0.0)])
def test_unipc_step_ignores_history_its_orders_do_not_read(ops, use_cfg, rescale):  # noqa: F811
    """NaN in the history buffers a step's orders do not read (all three at the loop's first step, prev_x0_2 at the
    second, where the corrector has order 1) leaves that step's outputs bit-identical."""
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    s = UniPCMultistepScheduler()
    s.set_timesteps(T_KERNEL)
    coeffs = torch.from_numpy(s.coeffs).cuda()
    n, h, w = 2, 64, 48
    g = torch.Generator().manual_seed(5)
    nan = lambda t: torch.full_like(t, float("nan"))  # noqa: E731
    for i, stale in ((0, ("last_sample", "prev_x0", "prev_x0_2")), (1, ("prev_x0_2",)), (6, ())):
        case = list(_step_case(s, i, n, 2 * n if use_cfg else n, h, w, g))
        clean = _run_kernel(ops, s, coeffs, i, 0, *case, use_cfg, rescale)
        names = {"last_sample": 2, "prev_x0": 3, "prev_x0_2": 4}
        for k in stale:
            case[names[k]] = nan(case[names[k]])
        dirty = _run_kernel(ops, s, coeffs, i, 0, *case, use_cfg, rescale)
        for k in ("latents", "last_sample", "prev_x0", "model_in"):
            assert torch.equal(clean[k], dirty[k]) and torch.isfinite(dirty[k]).all(), (i, k)
        if not stale:       # a step that reads them all does see the NaN
            case[4] = nan(case[4])
            assert torch.isnan(_run_kernel(ops, s, coeffs, i, 0, *case, use_cfg, rescale)["latents"]).all()


def _tiny_oracle_run(m, dev, dt, latents, pos, neg, ppool, npool, tid, T, karras, **kw):
    from unipc_ref import unipc_denoise_loop
    procs = [p for p in m.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    fn = lambda s, t, e, te, ti: m(s.to(dt), t, e, te, ti).to(torch.float16)  # noqa: E731
    return unipc_denoise_loop(fn, latents.to(dev), pos.to(dev, dt), neg.to(dev, dt), ppool.to(dev, dt),
                              npool.to(dev, dt), tid.to(dev), T, karras=karras, set_scale=set_scale, **kw)


@pytest.mark.parametrize("karras", [False, True])
def test_unipc_tiny_trajectory_matches_oracle(karras):
    """UniPC at T = 6, CFG 5.0, IP scale 0.8 gated off at the end, denoising_end 0.8: native eager and graph-replayed
    vs the fp32 CPU oracle with the bar of SURVEY section 7; the graph replay is bit-identical to the eager run and to a
    second replay."""
    from unipc_ref import UniPCRef, denoising_end_steps
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    native, ref32, eager16 = _make_pair(TINY, seed=31)
    T, n, lat = 6, 2, 32
    latents = prepare_latents(n, 4, lat, lat, [42, 43], 1.0)
    x = _inputs(TINY, n, lat, seed=33)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    kw = dict(guidance_scale=5.0, conditioning_scale=0.8, control_guidance_end=0.7, denoising_end=0.8)
    r = _tiny_oracle_run(ref32, "cpu", torch.float32, latents, *args, T, karras, **kw)
    e = _tiny_oracle_run(eager16, "cuda", torch.float16, latents, *args, T, karras, **kw)
    loop_steps = denoising_end_steps(UniPCRef(T, karras).timesteps.tolist(), 0.8)
    assert 1 < loop_steps < T
    outs = []
    for use_graph in (False, True, True):
        eng = DenoiseEngine(native, use_cuda_graph=use_graph, scheduler=UniPCMultistepScheduler(use_karras_sigmas=karras))
        calls = []
        o = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, control_guidance_end=0.7,
                    num_loop_steps=loop_steps, callback=lambda i, t, lt: calls.append(i))
        torch.cuda.synchronize()
        assert calls == list(range(loop_steps))
        e_nat, e_eag, mx = _errs(o, r, e)
        print(f"[unipc tiny karras={karras} graph={use_graph}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  "
              f"max|ref| {mx:.3e}")
        assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
        outs.append(o)
        if use_graph:
            o2 = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=0.8, control_guidance_end=0.7,
                         num_loop_steps=loop_steps)
            assert torch.equal(o, o2), "a second replay must reproduce the first"
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), "graph replay must equal the eager run"


def test_scheduler_swaps_and_batch_changes_bit_equal_to_fresh_pipelines():
    """Euler -> DPM (Karras) -> UniPC -> Euler on one pipeline, and n = 1 -> 3 -> 1 with UniPC: each call bit-identical
    to the same call on a fresh pipeline over the same UNet."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler, UniPCMultistepScheduler
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

    def uni():
        return UniPCMultistepScheduler.from_config(EulerDiscreteScheduler().config)
    pipe = StableDiffusionXLCustomPipeline(native)
    got = [call(pipe, 1)]
    pipe.scheduler = karras()
    got.append(call(pipe, 1))
    pipe.scheduler = uni()
    got += [call(pipe, 1), call(pipe, 3), call(pipe, 1)]
    pipe.scheduler = EulerDiscreteScheduler()
    got.append(call(pipe, 1))
    torch.cuda.synchronize()
    fresh = [call(StableDiffusionXLCustomPipeline(native), 1),
             call(StableDiffusionXLCustomPipeline(native, scheduler=karras()), 1),
             call(StableDiffusionXLCustomPipeline(native, scheduler=uni()), 1),
             call(StableDiffusionXLCustomPipeline(native, scheduler=uni()), 3)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], fresh[0]) and torch.equal(got[5], fresh[0])
    assert torch.equal(got[1], fresh[1])
    assert torch.equal(got[2], fresh[2]) and torch.equal(got[4], fresh[2])
    assert torch.equal(got[3], fresh[3])
    assert not torch.equal(got[0], got[2]) and not torch.equal(got[1], got[2])


def test_unipc_karras_sdxl_base_512_matches_oracle(sdxl_pair):  # noqa: F811
    """SDXL-base at 512^2: a 4-step UniPC Karras trajectory (CFG 5.0) through the CUDA-graph loop vs the CPU fp32
    oracle, bar of SURVEY section 7; then a graph-replayed 1024^2 10-step run comes out finite."""
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    cfg, native, ref, eager16 = sdxl_pair
    T, n, lat = 4, 1, 64
    latents = prepare_latents(n, 4, lat, lat, [42], 1.0)
    x = _inputs(cfg, n, lat, seed=13)
    args = (x["ehs"][n:], x["ehs"][:n], x["text_embeds"][n:], x["text_embeds"][:n], x["time_ids"][:n])
    with torch.no_grad():
        r4 = _tiny_oracle_run(ref, "cpu", torch.float32, latents, *args, T, True, guidance_scale=5.0)
        e4 = _tiny_oracle_run(eager16, "cuda", torch.float16, latents, *args, T, True, guidance_scale=5.0)
    eng = DenoiseEngine(native, scheduler=UniPCMultistepScheduler(use_karras_sigmas=True))
    o4 = eng.run(latents.pin_memory(), *args, T, guidance_scale=5.0, ip_scale=1.0)
    torch.cuda.synchronize()
    e_nat, e_eag, mx = _errs(o4, r4, e4)
    print(f"[UniPC Karras SDXL-base 512^2, 4 steps] native max|err| {e_nat:.3e}  eager-fp16 {e_eag:.3e}  "
          f"max|ref| {mx:.3e}")
    assert torch.isfinite(o4).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)

    lat = 128
    big = prepare_latents(n, 4, lat, lat, [7], 1.0)
    xb = _inputs(cfg, n, lat, seed=17)
    o = eng.run(big.pin_memory(), xb["ehs"][n:], xb["ehs"][:n], xb["text_embeds"][n:], xb["text_embeds"][:n],
                xb["time_ids"][:n], 10, guidance_scale=5.0, ip_scale=1.0)
    torch.cuda.synchronize()
    print(f"[UniPC Karras SDXL-base 1024^2, 10 steps] max|latent| {o.float().abs().max().item():.3e}")
    assert torch.isfinite(o).all()


def _graph_eager_and_restatement(monkeypatch, pipe, call, T, karras=False, guidance=5.0):
    """`call()` graph-replayed, then eagerly with every step's guided noise prediction and input latents recorded: the
    two runs must be bit-identical, and unipc_ref's steps applied to the recorded predictions must reproduce the eager
    run's latents at every step and at the end."""
    from unipc_ref import UniPCRef
    from imagharmony_b200 import ops as real_ops
    graph = call()
    assert pipe.engine.graphs_captured >= 1
    seen = []
    orig = real_ops.dpm_solver_step

    def record(noise_pred, latents, *a, **k):
        assert k.get("unipc") is not None, "a UniPC loop must run the UniPC step"
        seen.append((noise_pred.clone(), latents.clone()))
        return orig(noise_pred, latents, *a, **k)
    monkeypatch.setattr(real_ops, "dpm_solver_step", record)
    pipe.engine.use_cuda_graph = False
    eager = call()
    torch.cuda.synchronize()
    assert torch.isfinite(graph).all() and torch.equal(graph, eager), "graph replay must equal the eager run"
    assert len(seen) == T
    sched, x = UniPCRef(T, karras), seen[0][1]
    for noise_pred, latents in seen:
        assert torch.equal(x, latents)
        u, c = noise_pred.chunk(2)
        x = sched.step(u + guidance * (c - u), x)
    assert torch.equal(eager.to(x.device), x), (eager.float() - x.float()).abs().max()


def test_controlnet_loop_with_unipc_matches_restatement(monkeypatch):
    """StableDiffusionXLControlNetPipeline with UniPC at T = 5, CFG and a control window."""
    from test_controlnet_gpu import _call, _pipe
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    pipe = _pipe(seed=1)
    pipe.scheduler = UniPCMultistepScheduler()
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    kw = dict(control_guidance_start=0.2, control_guidance_end=0.8, controlnet_conditioning_scale=0.7)
    _graph_eager_and_restatement(monkeypatch, pipe, lambda: _call(pipe, img, T=5, **kw), 5)


def test_multi_controlnet_loop_with_unipc_matches_restatement(monkeypatch):
    """Multi-ControlNet (two nets with staggered guidance windows, so three step graphs) with UniPC at T = 6."""
    import test_multi_controlnet_gpu as mcn
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    pipe = mcn._pipe(seed=1)
    pipe.scheduler = UniPCMultistepScheduler()
    imgs = mcn._imgs(2, seed=2)
    kw = dict(controlnet_conditioning_scale=[0.9, 0.6], control_guidance_start=[0.0, 0.25],
              control_guidance_end=[0.5, 1.0], guidance_scale=5.0)
    _graph_eager_and_restatement(monkeypatch, pipe, lambda: mcn._call(pipe, imgs, T=6, **kw), 6)


@pytest.mark.parametrize("k", [1, 2])
def test_t2i_adapter_loop_with_unipc_matches_restatement(monkeypatch, k):
    """StableDiffusionXLAdapterPipeline (one adapter, and a MultiAdapter of two) with UniPC Karras at T = 5 and the
    features dropped halfway (adapter_conditioning_factor 0.5, so two step graphs)."""
    import test_t2i_adapter_gpu as t2i
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    pipe = t2i._pipe(seed=1, k=k)
    pipe.scheduler = UniPCMultistepScheduler(use_karras_sigmas=True)
    imgs = [torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(2 + j)) for j in range(k)]
    kw = dict(adapter_conditioning_factor=0.5, adapter_conditioning_scale=0.8 if k == 1 else [0.8, 0.3],
              guidance_scale=5.0)
    _graph_eager_and_restatement(monkeypatch, pipe, lambda: t2i._call(pipe, imgs[0] if k == 1 else imgs, T=5, **kw), 5,
                                 karras=True)
    assert pipe.engine.graphs_captured == 2                         # features on, features off


def test_ip_adapter_xl_generate_unipc_tiny_matches_oracle():
    """IPAdapterXL.generate over a TINY pipeline with UniPC Karras: the oracle pipeline from oracle/ parts with the
    same weights and the unipc_ref loop."""
    from unipc_ref import unipc_denoise_loop
    from imagharmony_b200.config import HARMONY_TINY, TINY
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
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
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config, use_karras_sigmas=True)
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
    want = unipc_denoise_loop(lambda s, t, e, a, b: ref_unet(s.float(), t, e, a, b).half(), lat, pos, neg, pp.float(),
                              npool.float(), tid, T, karras=True, guidance_scale=5.0)
    err = (out.float().cpu() - want.float()).abs().max().item()
    mx = want.float().abs().max().item()
    print(f"[IPAdapterXL.generate UniPC tiny] max|err| {err:.3e} max|ref| {mx:.3e}")
    assert err <= 2e-2 * mx, (err, mx)
