"""CPU tests of DPM-Solver++ 2M: the scheduler's tables and coefficient table against the restatement in
tests/dpm_ref.py and the known answers of SURVEY A.5, from_config, DenoiseEngine on the plain-PyTorch stand-in ops
(tests/fake_ops.py, tests/fake_ops_dpm.py) against the oracle loop, and the combinations that are refused."""
import numpy as np
import pytest
import torch

import fake_ops_dpm
from test_img2img_cpu import _pil_images
from test_inpaint_cpu import _embeds, _inpaint_pipe, _pil_masks
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def dpm(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_dpm.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_dpm, name))
    yield


@pytest.mark.parametrize("T,karras", [(20, False), (25, False), (20, True), (25, True)])
def test_tables_reproduce_known_answers(T, karras):
    from dpm_ref import KNOWN, dpm_tables
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    first_ts, last_ts, first_sig, last_sig = KNOWN[(T, karras)]
    assert s.timesteps.dtype == np.int64 and s.sigmas.dtype == np.float32
    assert s.timesteps.shape == (T,) and s.sigmas.shape == (T + 1,) and s.coeffs.shape == (T, 8)
    assert list(s.timesteps[:3]) == first_ts and list(s.timesteps[-2:]) == last_ts
    np.testing.assert_allclose(s.sigmas[:3], first_sig, atol=6e-6)
    np.testing.assert_allclose(s.sigmas[-3:], last_sig, atol=6e-6)
    assert s.sigmas[-1] == 0.0 and s.init_noise_sigma == 1.0 and s.order == 1
    ts, sig = dpm_tables(T, karras)
    assert np.array_equal(s.timesteps, ts) and np.array_equal(s.sigmas, sig)


def test_leading_spacing_uses_t_plus_one():
    """'leading' here divides by T + 1 (Euler divides by T): 1000 // 21 = 47 for T = 20, so 941 = 20 * 47 + 1."""
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
    d, e = DPMSolverMultistepScheduler(), EulerDiscreteScheduler()
    d.set_timesteps(20), e.set_timesteps(20)
    assert d.timesteps[0] == 941 and e.timesteps[0] == 951
    assert np.all(np.diff(d.timesteps) == -47)


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("T", [1, 2, 6, 20])
def test_coefficients_equal_per_step_diffusers_expressions(T, karras):
    """Each row of the coefficient table equals the diffusers expressions evaluated afresh at that step (dpm_ref), bit
    for bit; the first-order flag is set at index 0 and at T - 1 only (lower_order_final of final sigma 0)."""
    from dpm_ref import step_scalars
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    sig = torch.from_numpy(s.sigmas)
    for i in range(T):
        first = i == 0 or i == T - 1
        assert s.coeffs[i, 6] == (1.0 if first else 0.0) and s.coeffs[i, 7] == 0.0
        k = step_scalars(sig, i, not first)
        want = [k["sigma_s"], 1.0 / k["alpha_s"], k["ratio"], k["c"], k["c_half"], k.get("inv_r0", 0.0)]
        got = s.coeffs[i, :6].tolist()
        assert got == [float(v) for v in want], (i, got, want)
        assert np.isfinite(s.coeffs[i]).all()
    # the step to sigma 0: ratio 0 and c = -1, so the result is x0 exactly
    assert s.coeffs[T - 1, 2] == 0.0 and s.coeffs[T - 1, 3] == -1.0


def test_from_config_and_refused_fields():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
    cfg = EulerDiscreteScheduler().config
    assert cfg["timestep_spacing"] == "leading" and cfg["beta_end"] == 0.012 and cfg["use_karras_sigmas"] is False
    with pytest.raises(TypeError):
        cfg["use_karras_sigmas"] = True                                 # read-only
    k = DPMSolverMultistepScheduler.from_config(cfg, use_karras_sigmas=True)
    assert isinstance(k, DPMSolverMultistepScheduler) and k.use_karras_sigmas and k.kind == "dpmpp_2m_karras"
    plain = DPMSolverMultistepScheduler.from_config(cfg)
    assert not plain.use_karras_sigmas and plain.kind == "dpmpp_2m"
    k.set_timesteps(20)
    assert k.timesteps[0] == 999
    # round trip, and the fields that do not change the result
    again = DPMSolverMultistepScheduler.from_config(k.config, lower_order_final=False, euler_at_final=True)
    again.set_timesteps(20)
    assert np.array_equal(again.coeffs, k.coeffs)
    for bad in (dict(algorithm_type="dpmsolver"), dict(algorithm_type="sde-dpmsolver++"), dict(solver_order=3),
                dict(solver_order=1), dict(solver_type="heun"), dict(timestep_spacing="trailing"),
                dict(final_sigmas_type="sigma_min"), dict(thresholding=True), dict(prediction_type="v_prediction"),
                dict(use_lu_lambdas=True), dict(beta_schedule="linear"), dict(use_karas_sigmas=True)):
        with pytest.raises(IHError):
            DPMSolverMultistepScheduler.from_config(cfg, **bad)
    with pytest.raises(IHError):
        DPMSolverMultistepScheduler.from_config({**cfg, "timestep_spacing": "linspace"})


def _engine_vs_oracle(opts, karras, T=5, n=2, lat=8, seed=4):
    from dpm_ref import DPMSolverRef, denoising_end_steps, dpm_denoise_loop
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    native, ref = _build(TINY, seed)
    latents = prepare_latents(n, 4, lat, lat, [5, 6][:n], 1.0, dtype=torch.float32)
    _, ehs, te, tid = _inputs(TINY, n, lat, seed=9)
    procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    seen_ref, seen = [], []
    r = dpm_denoise_loop(lambda s, t, e, x, y: ref(s, t, e, x, y), latents.clone(), ehs[n:], ehs[:n], te[n:], te[:n],
                         tid[:n], T, karras=karras, set_scale=set_scale, conditioning_scale=0.8,
                         control_guidance_end=0.75, callback=lambda i, t, x: seen_ref.append((i, t, x.clone())),
                         callback_steps=2, **opts)
    eng = _fp32_engine(native)
    eng.scheduler = DPMSolverMultistepScheduler(use_karras_sigmas=karras)
    kw = dict(opts)
    loop_steps = denoising_end_steps(DPMSolverRef(T, karras).timesteps.tolist(), kw.pop("denoising_end", None))
    with _Empty32():
        o = eng.run(latents.clone(), ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], T, ip_scale=0.8,
                    control_guidance_end=0.75, num_loop_steps=loop_steps,
                    callback=lambda i, t, x: seen.append((i, float(t), x.clone())), callback_steps=2, **kw)
    return o, r, seen, seen_ref, loop_steps


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("opts", [
    dict(guidance_scale=5.0),
    dict(guidance_scale=1.0),
    dict(guidance_scale=5.0, guidance_rescale=0.7),
    dict(guidance_scale=5.0, denoising_end=0.6),
])
def test_engine_matches_oracle_loop(dpm, opts, karras):
    """DenoiseEngine with DPMSolverMultistepScheduler on the stand-in ops vs dpm_denoise_loop: CFG and no CFG, rescale,
    denoising_end (its last step stays second order), IP-scale gating and callback indices and timesteps."""
    o, r, seen, seen_ref, loop_steps = _engine_vs_oracle(opts, karras)
    if "denoising_end" in opts:
        assert 1 < loop_steps < 5
    assert torch.allclose(o, r, rtol=3e-4, atol=1e-3), (o - r).abs().max()
    assert [s[0] for s in seen] == [s[0] for s in seen_ref] == list(range(0, loop_steps, 2))
    assert [s[1] for s in seen] == [s[1] for s in seen_ref]
    for a, b in zip(seen, seen_ref):
        assert torch.allclose(a[2], b[2], rtol=3e-4, atol=1e-3)


def test_engine_second_order_matters(dpm):
    """The history is really used: forcing every step to first order (a table with every flag set) changes the result."""
    import imagharmony_b200.scheduler as S
    o, r, *_ = _engine_vs_oracle(dict(guidance_scale=5.0), False)
    orig = S.DPMSolverMultistepScheduler._coefficients

    def all_first(sigmas):
        c = orig(sigmas)
        c[:, 6] = 1.0
        return c
    S.DPMSolverMultistepScheduler._coefficients = staticmethod(all_first)
    try:
        o1, *_ = _engine_vs_oracle(dict(guidance_scale=5.0), False)
    finally:
        S.DPMSolverMultistepScheduler._coefficients = staticmethod(orig)
    assert (o1 - r).abs().max() > 100 * (o - r).abs().max()


def test_engine_refuses_resume_and_image_options(dpm):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    native, _ = _build(TINY, 4)
    _, ehs, te, tid = _inputs(TINY, 1, 8)
    args = (torch.zeros(1, 4, 8, 8), ehs[1:], ehs[:1], te[1:], te[:1], tid[:1], 4)
    ip = (torch.zeros(1, 4, 8, 8), torch.zeros(1, 4, 8, 8), torch.ones(1, 1, 8, 8))
    eng = _fp32_engine(native)
    eng.scheduler = DPMSolverMultistepScheduler()
    with _Empty32():
        for bad in (dict(begin_step=1), dict(inpaint=ip), dict(stop_after=2), dict(start_step=1)):
            with pytest.raises(IHError):
                eng.run(*args, **bad)
        assert eng.run(*args).shape == (1, 4, 8, 8)


def test_text_to_image_pipeline_takes_a_dpm_scheduler(dpm):
    """scheduler= and `pipe.scheduler = ...` both work; the engine integrates that object; the initial latents are the
    plain noise (init_noise_sigma 1); denoising_end counts DPM's timesteps (0.45 keeps 801, 601 of T = 4, Euler's
    schedule would keep 751 only)."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    emb = _embeds(1)
    common = dict(num_inference_steps=4, output_type="latent", height=64, width=64, **emb)
    dpm_s = DPMSolverMultistepScheduler.from_config(EulerDiscreteScheduler().config, use_karras_sigmas=True)
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    pipe2 = StableDiffusionXLCustomPipeline(pipe.unet, scheduler=dpm_s)
    assert pipe2.engine.scheduler is dpm_s
    noise = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(2))
    assert torch.equal(pipe2.prepare_latents(1, 4, 64, 64, torch.float16, "cpu", torch.Generator().manual_seed(2)),
                       noise.half())
    calls = []
    a = pipe2(generator=torch.Generator().manual_seed(1), callback=lambda i, t, x: calls.append((i, int(t))),
              **common).images
    assert calls == [(i, int(t)) for i, t in enumerate(dpm_s.timesteps)] and torch.isfinite(a.float()).all()
    e0 = pipe.engine
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)
    assert pipe.engine is not e0 and pipe.engine.scheduler is pipe.scheduler
    calls.clear()
    b = pipe(generator=torch.Generator().manual_seed(1), denoising_end=0.45,
             callback=lambda i, t, x: calls.append((i, int(t))), **common).images
    assert calls == [(0, 801), (1, 601)] and torch.isfinite(b.float()).all() and not torch.equal(a, b)


def test_img2img_and_inpaint_pipelines_refuse_dpm_before_any_work(dpm, monkeypatch):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    pipe = _inpaint_pipe()
    pipe.scheduler = DPMSolverMultistepScheduler()

    def no_work(*a, **k):
        raise AssertionError("work was done before the scheduler was checked")
    monkeypatch.setattr(pipe.vae_encoder, "encode_moments_nhwc", no_work)
    monkeypatch.setattr(pipe, "encode_prompt", no_work)
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    common = dict(prompt="lions", num_inference_steps=4, output_type="latent", generator=torch.Generator().manual_seed(0))
    with pytest.raises(IHError):
        pipe(image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=0.5, height=64, width=64, **common)
    with pytest.raises(IHError):
        StableDiffusionXLImg2ImgPipeline.__call__(pipe, image=_pil_images(1)[0], strength=0.5, **common)


def test_ip_adapter_xl_generate_through_dpm_pipeline(dpm):
    """IPAdapterXL(pipe with a DPM scheduler, ...).generate(...) with no change to ip_adapter.py."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=[7, 8],
                  output_type="latent", height=64, width=64)
    euler = ip_model.generate(**common)
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config, use_karras_sigmas=True)
    a = ip_model.generate(**common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    assert (a.float() - euler.float()).abs().max() > 1e-2
