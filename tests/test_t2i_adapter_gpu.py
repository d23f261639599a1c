"""GPU tests of the SDXL T2I-Adapter on the H100: the adapter forward (single and a 2-adapter MultiAdapter) against
the fp32 restatement of diffusers (tests/t2i_adapter_ref.py) at SDXL buckets, the feature injection bit-exact against
the torch fp16 expression, the SDXL-base UNet with features against the fp32 oracle UNet with diffusers' injection, the
graph-replayed TINY pipeline against the restated loop for every scheduler, graph replay against eager stepping, the
re-capture rules, and IPAdapterXL.generate on an adapter pipeline."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _bar(got, ref32, ref16):
    err = (got.float() - ref32).abs().max().item()
    e16 = (ref16.float() - ref32).abs().max().item()
    return err, max(2 * e16, 2e-3 * ref32.abs().max().item())


def _adapters(cfg, k, seed=0):
    """k native T2IAdapters (fp16, cuda) and their restatements in fp32 and fp16 (cuda)."""
    from imagharmony_b200.t2i_adapter import T2IAdapter
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from t2i_adapter_ref import T2IAdapterRef
    natives, refs = [], {torch.float32: [], torch.float16: []}
    with torch.device("meta"):
        shapes = shapes_of(T2IAdapterRef(cfg))
    for j in range(k):
        sd = random_state_dict(shapes, seed + 7 * j, device="cuda")
        natives.append(T2IAdapter.from_state_dict(cfg, sd))
        for dt in refs:
            r = T2IAdapterRef(cfg)
            r.load_state_dict({n: v.float() for n, v in sd.items()})
            refs[dt].append(r.to("cuda", dt).eval())
    return natives, refs


FORWARD_CASES = [(h, w, n, k) for h, w in ((1024, 1024), (832, 1216), (1536, 640)) for n in (1, 4) for k in (1, 2)]


@pytest.mark.parametrize("height,width,n,k", FORWARD_CASES,
                         ids=[f"{h}x{w}-n{n}-k{k}" for h, w, n, k in FORWARD_CASES])
def test_adapter_forward_matches_reference(height, width, n, k):
    from imagharmony_b200.config import SDXL_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import MultiAdapter
    from t2i_adapter_ref import multi_adapter_ref
    natives, refs = _adapters(SDXL_T2I_ADAPTER, k, seed=3)
    g = torch.Generator().manual_seed(height + n + k)
    xs = [torch.rand(n, 3, height, width, generator=g).half().cuda() for _ in range(k)]
    weights = [0.7, 0.45][:k]
    with torch.no_grad():
        if k == 1:
            got = natives[0](xs[0])
            want = {dt: r[0](xs[0].to(dt)) for dt, r in refs.items()}
        else:
            got = MultiAdapter(natives)(xs, weights)
            want = {dt: multi_adapter_ref(r, [x.to(dt) for x in xs], weights) for dt, r in refs.items()}
    for i, (gf, r32, r16) in enumerate(zip(got, want[torch.float32], want[torch.float16])):
        err, lim = _bar(gf.permute(0, 3, 1, 2), r32, r16)
        assert err <= lim, (i, err, lim)


@pytest.mark.parametrize("cfg", [True, False])
def test_injection_bit_exact_sdxl_shapes(cfg):
    """At 1024^2 (the 4 injection points of SDXL-base), each CFG half: fp16(skip + fp16(v * s)), in place."""
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.unet import adapter_targets
    g = torch.Generator().manual_seed(1)
    n = 2
    halves = 2 if cfg else 1
    s = 0.8
    scale = torch.full((2,), s, dtype=torch.float32, device="cuda")
    for h, w, c in adapter_targets(SDXL_BASE, 128, 128):
        skip = (torch.randn(halves * n, h, w, c, generator=g) * 3).half().cuda()
        feat = (torch.randn(n, h, w, c, generator=g) * 2).half().cuda()
        want = (skip.float() + (feat * s).float().repeat(halves, 1, 1, 1)).half()      # diffusers: v * s, then +
        ptr = skip.data_ptr()
        ops.controlnet_add_residuals([skip] * halves, [feat] * halves, scale, [r * n * h * w for r in range(halves)])
        torch.cuda.synchronize()
        assert skip.data_ptr() == ptr and torch.equal(skip, want), (h, w, c)


def test_sdxl_unet_with_features_matches_oracle():
    """SDXL-base at 1024^2, CFG batch: the native UNet with adapter_residuals against the fp32 (and fp16) restatement
    with diffusers' down_intrablock_additional_residuals."""
    from oracle import adapter_ref as A
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.unet import UNet2DConditionModel, adapter_targets
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from t2i_adapter_ref import UNetAdapterRef
    with torch.device("meta"):
        shapes = shapes_of(UNetAdapterRef(SDXL_BASE))
    usd = random_state_dict(shapes, 5, device="cuda")
    unet = UNet2DConditionModel.from_state_dict(SDXL_BASE, usd)
    g = torch.Generator().manual_seed(2)
    sample = torch.randn(2, 4, 128, 128, generator=g).half().cuda()
    ehs = torch.randn(2, 81, 2048, generator=g).half().cuda()
    te = torch.randn(2, 1280, generator=g).half().cuda()
    tid = torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * 2).cuda()
    feats = [(torch.randn(1, h, w, c, generator=g) * 0.5).half().cuda() for h, w, c in adapter_targets(SDXL_BASE, 128, 128)]
    s = 0.9
    with torch.no_grad():
        got = unet(sample, torch.full((2,), 501.0, device="cuda"), ehs, te, tid,
                   adapter_residuals=(feats, torch.full((2,), s, device="cuda")))
        del unet
        ref = {}
        for dt in (torch.float32, torch.float16):
            ru = UNetAdapterRef(SDXL_BASE)
            ru.load_state_dict({k: v.float() for k, v in usd.items()})
            for p in A.install_processors(ru, SDXL_BASE).values():
                for q in p.parameters():
                    q.data.zero_()
            ru = ru.to("cuda", dt).eval()
            state = [torch.cat([(f * s).permute(0, 3, 1, 2)] * 2).to(dt) for f in feats]
            ref[dt] = ru(sample.to(dt), 501.0, ehs.to(dt), te.to(dt), tid.to(dt),
                         down_intrablock_additional_residuals=state).float()
            del ru
            torch.cuda.empty_cache()
    err, lim = _bar(got, ref[torch.float32], ref[torch.float16])
    assert err <= lim, (err, lim)


# ---------------------------------------------------------------------------------------------------------------------
# the TINY pipeline
# ---------------------------------------------------------------------------------------------------------------------
def _pipe(seed=0, k=1, cfg_u=None):
    from imagharmony_b200.config import TINY, TINY_T2I_ADAPTER
    from ip_adapter.custom_pipelines import StableDiffusionXLAdapterPipeline
    return StableDiffusionXLAdapterPipeline.from_random(cfg_u or TINY, [TINY_T2I_ADAPTER] * k if k > 1 else TINY_T2I_ADAPTER,
                                                        seed=seed)


def _emb(pipe, n=1):
    gen = torch.Generator("cpu").manual_seed(9)
    D, P = pipe.unet.config.cross_attention_dim, pipe.unet.config.pooled_embed_dim
    return dict(prompt_embeds=torch.randn(n, 77, D, generator=gen).half(),
                negative_prompt_embeds=torch.randn(n, 77, D, generator=gen).half(),
                pooled_prompt_embeds=torch.randn(n, P, generator=gen).half(),
                negative_pooled_prompt_embeds=torch.randn(n, P, generator=gen).half())


def _call(pipe, img, T=4, seed=3, **kw):
    g = torch.Generator("cuda").manual_seed(seed)
    return pipe(image=img, num_inference_steps=T, generator=g, output_type="latent", **_emb(pipe), **kw).images


def _set_scheduler(pipe, sched):
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    pipe.scheduler = {"euler": EulerDiscreteScheduler(), "euler_a": EulerAncestralDiscreteScheduler(),
                      "dpm": DPMSolverMultistepScheduler(use_karras_sigmas=True)}[sched]


SCHEDULERS = ["euler", "euler_a", "dpm"]
OPTS = [dict(), dict(adapter_conditioning_factor=0.5, adapter_conditioning_scale=0.7),
        dict(guidance_scale=1.0, denoising_end=0.8)]


@pytest.mark.parametrize("sched", SCHEDULERS)
@pytest.mark.parametrize("opts", OPTS)
def test_tiny_trajectory_matches_restated_loop(sched, opts):
    from dpm_ref import denoising_end_steps as dpm_end_steps, dpm_denoise_loop, dpm_tables
    from euler_a_ref import euler_a_denoise_loop
    from imagharmony_b200.config import TINY, TINY_T2I_ADAPTER
    from oracle import adapter_ref as A
    from oracle.scheduler_ref import denoise_loop, denoising_end_steps
    from t2i_adapter_ref import T2IAdapterRef, UNetAdapterRef, adapter_state_ref, adapter_unet_fn
    pipe = _pipe(seed=2)
    _set_scheduler(pipe, sched)
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    T = 4
    got = _call(pipe, img, T=T, **opts).float()
    guidance = opts.get("guidance_scale", 5.0)
    dend = opts.get("denoising_end")
    if sched == "dpm":
        loop_T = dpm_end_steps(dpm_tables(T, karras=True)[0].tolist(), dend)
    else:
        loop_T = denoising_end_steps(T, dend)
    e = _emb(pipe)
    usd = {k: v for k, v in pipe.unet.state_dict().items() if "processor" not in k}
    outs = {}
    with torch.no_grad():
        for dt in (torch.float32, torch.float16):
            ru = UNetAdapterRef(TINY)
            ru.load_state_dict({k: v.float() for k, v in usd.items()})
            for p in A.install_processors(ru, TINY).values():
                for q in p.parameters():
                    q.data.zero_()
            ru = ru.to("cuda", dt).eval()
            ra = T2IAdapterRef(TINY_T2I_ADAPTER)
            ra.load_state_dict({k: v.float() for k, v in pipe.adapter.state_dict().items()})
            ra = ra.to("cuda", dt).eval()
            feats = ra(img.half().cuda().to(dt))
            state = adapter_state_ref(feats, opts.get("adapter_conditioning_scale", 1.0), 1, guidance > 1.0)
            fn = adapter_unet_fn(ru, state, loop_T, opts.get("adapter_conditioning_factor", 1.0))
            g = torch.Generator("cuda").manual_seed(3)
            ins = 1.0 if sched == "dpm" else pipe.scheduler.init_noise_sigma
            lat0 = (torch.randn((1, 4, 16, 16), generator=g, device="cuda") * ins).half().to(dt)
            tid = torch.tensor([[128., 128, 0, 0, 128, 128]], device="cuda", dtype=dt)
            args = (fn, lat0, e["prompt_embeds"].cuda().to(dt), e["negative_prompt_embeds"].cuda().to(dt),
                    e["pooled_prompt_embeds"].cuda().to(dt), e["negative_pooled_prompt_embeds"].cuda().to(dt), tid, T)
            common = dict(guidance_scale=guidance, denoising_end=dend)
            if sched == "euler":
                outs[dt] = denoise_loop(*args, **common).float()
            elif sched == "euler_a":
                outs[dt] = euler_a_denoise_loop(*args, generator=g, **common).float()
            else:
                outs[dt] = dpm_denoise_loop(*args, karras=True, **common).float()
    err, lim = _bar(got, outs[torch.float32], outs[torch.float16])
    assert err <= max(lim, 2e-2 * outs[torch.float32].abs().max().item()), (err, lim)


@pytest.mark.parametrize("sched", SCHEDULERS)
@pytest.mark.parametrize("k", [1, 2])
def test_graph_replay_bit_identical_to_eager(sched, k):
    pipe = _pipe(seed=1, k=k)
    _set_scheduler(pipe, sched)
    imgs = [torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(2 + j)) for j in range(k)]
    opts = dict(adapter_conditioning_factor=0.5, adapter_conditioning_scale=0.8 if k == 1 else [0.8, 0.3])
    graph = _call(pipe, imgs[0] if k == 1 else imgs, **opts)
    assert pipe.engine.graphs_captured == 2                         # features on, features off
    pipe.engine.use_cuda_graph = False
    eager = _call(pipe, imgs[0] if k == 1 else imgs, **opts)
    assert torch.isfinite(graph).all() and torch.equal(graph, eager)


def test_scale_and_image_change_do_not_recapture():
    from ip_adapter.custom_pipelines import StableDiffusionXLAdapterPipeline
    pipe = _pipe(seed=3)
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    img2 = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(6))
    a = _call(pipe, img, adapter_conditioning_scale=1.0)
    n = pipe.engine.graphs_captured
    b = _call(pipe, img2, adapter_conditioning_scale=0.4)
    assert pipe.engine.graphs_captured == n and not torch.equal(a, b)
    fresh = StableDiffusionXLAdapterPipeline(pipe.unet, pipe.adapter)
    assert torch.equal(b, _call(fresh, img2, adapter_conditioning_scale=0.4))
    zero = _call(pipe, img, adapter_conditioning_scale=0.0)
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    t2i = StableDiffusionXLCustomPipeline(pipe.unet)
    want = t2i(height=128, width=128, num_inference_steps=4, generator=torch.Generator("cuda").manual_seed(3),
               output_type="latent", **_emb(pipe)).images
    assert torch.equal(zero, want)                                 # fp16(x + fp16(v * 0)) = x


def test_ip_adapter_generate_with_sketch():
    from PIL import Image
    from ip_adapter.ip_adapter import IPAdapterXL
    pipe = _pipe(seed=4)
    ip = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4)
    emb = torch.randn(1, ip._clip_dim(), generator=torch.Generator().manual_seed(0))
    sketch = Image.fromarray((torch.rand(128, 128, 3, generator=torch.Generator().manual_seed(1)) * 255).byte().numpy())
    out = ip.generate(clip_image_embeds=emb, num_samples=2, seed=0, num_inference_steps=3, image=[sketch] * 2,
                      adapter_conditioning_scale=0.8, output_type="latent")
    assert out.shape == (2, 4, 16, 16) and torch.isfinite(out.float()).all()
