"""CPU tests of Euler Ancestral: the scheduler's tables and coefficient table against Euler's and the restatement in
tests/euler_a_ref.py, from_config, DenoiseEngine on the plain-PyTorch stand-in ops (tests/fake_ops.py,
tests/fake_ops_euler_a.py) against the oracle loop -- including the generator state after the per-step draws -- and
the three pipelines end to end with diffusers' RNG order of preparation and steps."""
import numpy as np
import pytest
import torch

import fake_ops_euler_a
from test_img2img_cpu import _img2img_pipe, _oracle_for, _pil_images, i2i  # noqa: F401  (fixture)
from test_inpaint_cpu import _embeds, _inpaint_pipe, _pil_masks, inp  # noqa: F401  (fixture)
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def ea(inp, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_euler_a.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_euler_a, name))
    yield


@pytest.mark.parametrize("T", [4, 20, 30, 50])
def test_tables_equal_euler(T):
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler, EulerDiscreteScheduler
    a, e = EulerAncestralDiscreteScheduler(), EulerDiscreteScheduler()
    sa, se = a.set_timesteps(T), e.set_timesteps(T)
    assert np.array_equal(sa.timesteps, se.timesteps) and np.array_equal(sa.sigmas, se.sigmas)
    assert a.init_noise_sigma == e.init_noise_sigma and a.order == 1 and a.kind == "euler_a"
    assert a.coeffs.shape == (T, 8) and a.coeffs.dtype == np.float32
    assert a.img2img_begin_index(T, 0.6) == e.img2img_begin_index(T, 0.6)
    assert a.add_noise_sigma(3) == e.add_noise_sigma(3)


@pytest.mark.parametrize("T", [1, 4, 20, 50])
def test_coefficients_equal_diffusers_expressions(T):
    """Each row equals diffusers' step() / scale_model_input() scalars evaluated afresh (euler_a_ref's sigmas on the
    CPU), bit for bit; the last row has sigma_up = 0 and dt = -sigma."""
    from euler_a_ref import EulerAncestralRef
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    s = EulerAncestralDiscreteScheduler()
    s.set_timesteps(T)
    sig = EulerAncestralRef(T).sigmas
    for i in range(T):
        sf, st = sig[i], sig[i + 1]
        up = (st**2 * (sf**2 - st**2) / sf**2) ** 0.5
        down = (st**2 - up**2) ** 0.5
        want = [sf, 1.0 / sf, down - sf, up, 1.0 / ((st**2 + 1) ** 0.5), st.to(torch.float16),
                1.0 / ((sf**2 + 1) ** 0.5), 0.0]
        assert s.coeffs[i].tolist() == [float(v) for v in want], i
        assert np.isfinite(s.coeffs[i]).all()
    assert s.coeffs[T - 1, 3] == 0.0 and s.coeffs[T - 1, 2] == -s.coeffs[T - 1, 0]
    if T > 1:
        assert (s.coeffs[:-1, 3] > 0).all()
        assert np.array_equal(s.coeffs[1:, 6], s.coeffs[:-1, 4])     # a resumed first input equals a step's output


def test_from_config_and_refused_fields():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    e_cfg = EulerDiscreteScheduler().config
    d_cfg = DPMSolverMultistepScheduler().config
    for cfg in (e_cfg, d_cfg):
        a = EulerAncestralDiscreteScheduler.from_config(cfg)
        assert isinstance(a, EulerAncestralDiscreteScheduler) and a.kind == "euler_a"
        a.set_timesteps(20)
        assert a.timesteps[0] == 951
    a = EulerAncestralDiscreteScheduler.from_config(e_cfg, steps_offset=1)
    with pytest.raises(TypeError):
        a.config["steps_offset"] = 0                                       # read-only
    again = EulerAncestralDiscreteScheduler.from_config(a.config)
    again.set_timesteps(20), a.set_timesteps(20)
    assert np.array_equal(again.coeffs, a.coeffs)
    for bad in (dict(prediction_type="v_prediction"), dict(timestep_spacing="trailing"), dict(beta_schedule="linear"),
                dict(use_karras_sigmas=True), dict(rescale_betas_zero_snr=True), dict(solver_order=2)):
        with pytest.raises(IHError):
            EulerAncestralDiscreteScheduler.from_config(e_cfg, **bad)
    with pytest.raises(IHError):
        EulerAncestralDiscreteScheduler.from_config(DPMSolverMultistepScheduler(use_karras_sigmas=True).config)
    with pytest.raises(IHError):
        EulerAncestralDiscreteScheduler.from_config({**e_cfg, "timestep_spacing": "linspace"})


def _gens(list_gen, n=2, base=21):
    return ([torch.Generator().manual_seed(base + k) for k in range(n)] if list_gen
            else torch.Generator().manual_seed(base))


def _same_state(a, b):
    a, b = (a if isinstance(a, list) else [a]), (b if isinstance(b, list) else [b])
    return all(torch.equal(x.get_state(), y.get_state()) for x, y in zip(a, b))


def _engine_vs_oracle(opts, T=4, n=2, lat=8, seed=4, list_gen=False, begin=0, inpaint=False, gen_base=21):
    from euler_a_ref import euler_a_denoise_loop
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from oracle.scheduler_ref import euler_tables, prepare_latents
    native, ref = _build(TINY, seed)
    ts, _, ins = euler_tables(T)
    latents = prepare_latents(n, 4, lat, lat, [5, 6][:n], ins, dtype=torch.float32)
    _, ehs, te, tid = _inputs(TINY, n, lat, seed=9)
    procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]
    blend = None
    if inpaint:
        g = torch.Generator().manual_seed(3)
        blend = (torch.randn(n, 4, lat, lat, generator=g), torch.randn(n, 4, lat, lat, generator=g),
                 (torch.rand(n, 1, lat, lat, generator=g) > 0.5).float())

    def set_scale(s):
        for p in procs:
            p.scale = s
    seen_ref, seen = [], []
    g_ref = _gens(list_gen, n, gen_base)
    r = euler_a_denoise_loop(lambda s, t, e, x, y: ref(s, t, e, x, y), latents.clone(), ehs[n:], ehs[:n], te[n:],
                             te[:n], tid[:n], T, generator=g_ref, set_scale=set_scale, conditioning_scale=0.8,
                             control_guidance_end=0.75, callback=lambda i, t, x: seen_ref.append((i, t, x.clone())),
                             callback_steps=2, begin=begin, blend=blend, **opts)
    eng = _fp32_engine(native)
    eng.scheduler = EulerAncestralDiscreteScheduler()
    kw = dict(opts)
    de = kw.pop("denoising_end", None)
    loop_end = T
    if de is not None:
        loop_end = begin + sum(1 for t in ts[begin:] if t >= int(round(1000 - de * 1000)))
    g_eng = _gens(list_gen, n, gen_base)
    with _Empty32():
        o = eng.run(latents.clone(), ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], T, ip_scale=0.8,
                    control_guidance_end=0.75, num_loop_steps=loop_end, begin_step=begin, inpaint=blend,
                    callback=lambda i, t, x: seen.append((i, float(t), x.clone())), callback_steps=2,
                    generator=g_eng, **kw)
    return o, r, seen, seen_ref, g_eng, g_ref, loop_end - begin


@pytest.mark.parametrize("opts,kw", [
    (dict(guidance_scale=5.0), dict()),
    (dict(guidance_scale=1.0), dict(list_gen=True)),
    (dict(guidance_scale=5.0, guidance_rescale=0.7), dict()),
    (dict(guidance_scale=5.0, denoising_end=0.6), dict(list_gen=True)),
    (dict(guidance_scale=5.0), dict(begin=1)),
    (dict(guidance_scale=5.0, denoising_end=0.8), dict(begin=1, inpaint=True)),
    (dict(guidance_scale=1.0), dict(inpaint=True, list_gen=True)),
])
def test_engine_matches_oracle_loop(ea, opts, kw):
    """DenoiseEngine with EulerAncestralDiscreteScheduler on the stand-in ops vs euler_a_denoise_loop: CFG on / off,
    rescale, denoising_end, IP-scale gating, callbacks, begin_step and inpaint; the generator(s) end in the state of
    the oracle's draws (one per executed step)."""
    o, r, seen, seen_ref, g_eng, g_ref, n_loop = _engine_vs_oracle(opts, **kw)
    assert n_loop >= 2
    assert torch.allclose(o, r, rtol=3e-4, atol=1e-3), (o - r).abs().max()
    assert [s[0] for s in seen] == [s[0] for s in seen_ref] == list(range(0, n_loop, 2))
    assert [s[1] for s in seen] == [s[1] for s in seen_ref]
    for a, b in zip(seen, seen_ref):
        assert torch.allclose(a[2], b[2], rtol=3e-4, atol=1e-3)
    assert _same_state(g_eng, g_ref)


def test_engine_noise_matters(ea):
    """The per-step noise is really added: another seed gives another result."""
    o, *_ = _engine_vs_oracle(dict(guidance_scale=5.0))
    o2, *_ = _engine_vs_oracle(dict(guidance_scale=5.0), gen_base=40)
    assert (o - o2).abs().max() > 1e-2


def _resume_args(n=1, lat=8):
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    native, _ = _build(TINY, 4)
    _, ehs, te, tid = _inputs(TINY, n, lat)
    latents = torch.randn(n, 4, lat, lat, generator=torch.Generator().manual_seed(8))
    eng = _fp32_engine(native)
    eng.scheduler = EulerAncestralDiscreteScheduler()
    return eng, (ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], 5), latents


@pytest.mark.parametrize("list_gen", [False, True])
def test_stop_and_resume_reproduce_the_uninterrupted_run(ea, list_gen):
    """stop_after=k then start_step=k on the same, continuing generator equals the uninterrupted run; the stopped call
    draws k noises only."""
    from euler_a_ref import randn_tensor_ref
    n = 2
    eng, args, latents = _resume_args(n)
    with _Empty32():
        g = _gens(list_gen, n)
        full = eng.run(latents, *args, generator=g)
        g1 = _gens(list_gen, n)
        part = eng.run(latents, *args, stop_after=2, generator=g1)
        g_ref = _gens(list_gen, n)
        for _ in range(2):
            randn_tensor_ref((n, 4, 8, 8), g_ref, "cpu", torch.float16)
        assert _same_state(g1, g_ref)
        rest = eng.run(part, *args, start_step=2, generator=g1)
    assert torch.equal(rest, full) and _same_state(g1, g)


def test_generator_none_draws_from_the_default_generator(ea):
    eng, args, latents = _resume_args()
    with _Empty32():
        torch.manual_seed(5)
        a = eng.run(latents, *args)
        torch.manual_seed(5)
        b = eng.run(latents, *args)
        c = eng.run(latents, *args)
    assert torch.equal(a, b) and not torch.equal(a, c)


def test_generator_list_length_must_match_the_batch(ea):
    from imagharmony_b200._lib import IHError
    eng, args, latents = _resume_args(2)
    with _Empty32(), pytest.raises(IHError):
        eng.run(latents, *args, generator=_gens(True, 3))


@pytest.mark.parametrize("list_gen", [False, True])
def test_text_to_image_pipeline_matches_oracle(ea, list_gen):
    """pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(...): the start latents are drawn and scaled as
    with Euler, then every step draws its noise from the same generator(s) -- the pipeline vs the oracle chain."""
    from euler_a_ref import EulerAncestralRef, euler_a_denoise_loop, randn_tensor_ref
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    ref = _oracle_for_unet(pipe)
    emb = _embeds(2)
    T = 4
    seen = []
    out = pipe(generator=_gens(list_gen), num_inference_steps=T, output_type="latent", height=64, width=64,
               callback=lambda i, t, x: seen.append((i, int(t))), **emb).images
    g = _gens(list_gen)
    lat = (randn_tensor_ref((2, 4, 8, 8), g, "cpu", torch.float32) * EulerAncestralRef(T).init_noise_sigma).half()
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    r = euler_a_denoise_loop(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), lat,
                             emb["prompt_embeds"].float(), emb["negative_prompt_embeds"].float(),
                             emb["pooled_prompt_embeds"].float(), emb["negative_pooled_prompt_embeds"].float(), tid, T,
                             generator=g)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (2, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    assert seen == [(i, int(t)) for i, t in enumerate(pipe.scheduler.timesteps)]


def _oracle_for_unet(pipe):
    from imagharmony_b200.config import TINY
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    ref = UNetRef(TINY)
    A.install_processors(ref, TINY)
    ref.load_state_dict({k: v.float() for k, v in pipe.unet.state_dict().items()})
    return ref.eval()


@pytest.mark.parametrize("list_gen", [False, True])
def test_img2img_pipeline_matches_oracle(ea, list_gen):
    """Image-to-image with Euler A: posterior eps, then noise (C.18), then one draw per executed step."""
    from PIL import Image
    from euler_a_ref import euler_a_denoise_loop
    from img2img_ref import img2img_timesteps, prepare_img2img_latents
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from oracle.scheduler_ref import euler_tables
    pipe = _img2img_pipe()
    pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    ref, procs, venc = _oracle_for(pipe)
    imgs, emb = _pil_images(2), _embeds(4)
    T, strength = 5, 0.6

    def gens():
        return [torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)] if list_gen else torch.Generator().manual_seed(1)
    out = pipe(image=imgs, strength=strength, num_inference_steps=T, generator=gens(), output_type="latent",
               **emb).images
    pix = np.stack([np.array(im.resize((64, 64), resample=Image.LANCZOS)).astype(np.float32) / 255.0 for im in imgs])
    pix = torch.from_numpy(pix).permute(0, 3, 1, 2) * 2.0 - 1.0
    t_start, _ = img2img_timesteps(T, strength)
    g = gens()
    with torch.no_grad():
        lat = prepare_img2img_latents(venc.encode, pix, 4, g, float(euler_tables(T)[1][t_start]),
                                      TINY_VAE.scaling_factor)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    r = euler_a_denoise_loop(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), lat,
                             emb["prompt_embeds"].float(), emb["negative_prompt_embeds"].float(),
                             emb["pooled_prompt_embeds"].float(), emb["negative_pooled_prompt_embeds"].float(), tid, T,
                             generator=g, begin=t_start)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (4, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)


@pytest.mark.parametrize("opts", [
    dict(strength=0.5, n_img=2, n_masks=1, list_gen=True),
    dict(strength=1.0, n_img=1, n_masks=2, list_gen=False, denoising_end=0.6),
])
def test_inpaint_pipeline_matches_oracle(ea, opts):
    """Inpainting with Euler A: posterior eps, noise (C.19), the unused masked-image posterior draw (C.31), then one
    draw per executed step; the blend after every step."""
    from PIL import Image
    from euler_a_ref import euler_a_denoise_loop, masked_image_draw_ref
    from img2img_ref import img2img_timesteps
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from inpaint_ref import mask_latents_ref, prepare_inpaint_latents, preprocess_mask_ref
    opts = dict(opts)
    n_img, n_masks, list_gen = opts.pop("n_img"), opts.pop("n_masks"), opts.pop("list_gen")
    strength = opts.pop("strength")
    pipe = _inpaint_pipe()
    pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    ref, procs, venc = _oracle_for(pipe)
    imgs, masks, emb = _pil_images(n_img), _pil_masks(n_masks), _embeds(4)
    T = 5

    def gens():
        return [torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)] if list_gen else torch.Generator().manual_seed(1)
    out = pipe(image=imgs if n_img > 1 else imgs[0], mask_image=masks if n_masks > 1 else masks[0], strength=strength,
               num_inference_steps=T, height=64, width=64, generator=gens(), output_type="latent", **opts,
               **emb).images
    pix = np.stack([np.array(im.resize((64, 64), resample=Image.LANCZOS)).astype(np.float32) / 255.0 for im in imgs])
    pix = torch.from_numpy(pix).permute(0, 3, 1, 2) * 2.0 - 1.0
    t_start, _ = img2img_timesteps(T, strength)
    g = gens()
    with torch.no_grad():
        lat, img_lat, noise = prepare_inpaint_latents(venc.encode, pix, 4, g, t_start, T, strength,
                                                      TINY_VAE.scaling_factor)
    masked_image_draw_ref(max(n_img, n_masks), (4, 8, 8), g)
    mask = mask_latents_ref(preprocess_mask_ref(masks, 64, 64), 4, 64, 64)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    r = euler_a_denoise_loop(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), lat,
                             emb["prompt_embeds"].float(), emb["negative_prompt_embeds"].float(),
                             emb["pooled_prompt_embeds"].float(), emb["negative_pooled_prompt_embeds"].float(), tid, T,
                             generator=g, guidance_scale=7.5, begin=t_start, blend=(img_lat, noise, mask), **opts)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (4, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    keep = (mask == 0).expand_as(r)
    assert (out.float() - img_lat.float())[keep].abs().max() <= 2e-2 * mx


def test_ip_adapter_xl_generate_through_euler_a_pipeline(ea):
    """IPAdapterXL(pipe with an Euler A scheduler, ...).generate(...) with no change to ip_adapter.py: seeded, the
    result repeats, and it differs from Euler's."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=42,
                  output_type="latent", height=64, width=64)
    euler = ip_model.generate(**common)
    pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    a, b = ip_model.generate(**common), ip_model.generate(**common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all() and torch.equal(a, b)
    assert (a.float() - euler.float()).abs().max() > 1e-2
