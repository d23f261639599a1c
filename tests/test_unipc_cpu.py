"""CPU tests of UniPC: the scheduler's tables, order schedule and coefficient table against the restatement in
tests/unipc_ref.py and the known answers of SURVEY A.9, from_config, DenoiseEngine on the plain-PyTorch stand-in ops
(tests/fake_ops.py, tests/fake_ops_unipc.py) against the oracle loop, the combinations that are refused, and the
C entry point's argument checks."""
import ctypes

import numpy as np
import pytest
import torch

import fake_ops_unipc
from test_img2img_cpu import _pil_images
from test_inpaint_cpu import _embeds, _inpaint_pipe, _pil_masks
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def unipc(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_unipc.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_unipc, name))
    yield


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("T", [10, 20, 25])
def test_tables_reproduce_known_answers(T, karras):
    from dpm_ref import dpm_tables
    from unipc_ref import KNOWN
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    s = UniPCMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    first_ts, last_ts, first_sig, last_sig = KNOWN[(T, karras)]
    assert s.timesteps.dtype == np.int64 and s.sigmas.dtype == np.float32
    assert s.timesteps.shape == (T,) and s.sigmas.shape == (T + 1,) and s.coeffs.shape == (T, 16)
    assert list(s.timesteps[:3]) == first_ts and list(s.timesteps[-2:]) == last_ts
    np.testing.assert_allclose(s.sigmas[:3], first_sig, atol=6e-6)
    np.testing.assert_allclose(s.sigmas[-3:], last_sig, atol=6e-6)
    assert s.sigmas[-1] == 0.0 and s.init_noise_sigma == 1.0 and s.order == 1
    ts, sig = dpm_tables(T, karras)
    assert np.array_equal(s.timesteps, ts) and np.array_equal(s.sigmas, sig)


@pytest.mark.parametrize("T", [1, 2, 3, 5, 20])
def test_order_schedule(T):
    """No corrector at the loop's first step, c(i) = p(i - 1) after it, predictor order 1 at the first and the last
    index, 2 in between; the table's columns carry the schedule of a loop from index 0, and a later loop start lowers
    the orders as the kernel's rule min(table, i - b + 1) / min(table, i - b) does."""
    from unipc_ref import orders
    from imagharmony_b200.scheduler import UniPCMultistepScheduler, unipc_orders
    p, c = orders(T)
    assert (p, c) == unipc_orders(T)
    assert c[0] == 0 and p[0] == 1 and p[T - 1] == 1
    assert all(c[i] == p[i - 1] for i in range(1, T))
    assert all(p[i] == 2 for i in range(1, T - 1))
    s = UniPCMultistepScheduler()
    s.set_timesteps(T)
    assert s.coeffs[:, 5].tolist() == p and s.coeffs[:, 11].tolist() == c
    for b in range(T):
        pb, cb = orders(T, b)
        assert pb[b:] == [min(p[i], i - b + 1) for i in range(b, T)]
        assert cb[b:] == [min(c[i], i - b) if i > b else 0 for i in range(b, T)]


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("T", [1, 2, 3, 6, 20])
def test_coefficients_equal_per_step_diffusers_expressions(T, karras):
    """Each row equals the diffusers expressions evaluated afresh at that step (unipc_ref.step_scalars, including the
    linalg.solve of the order-2 corrector and the fp16 rounding of its rhos), bit for bit; scalars of an order the row
    does not use are 0."""
    from unipc_ref import orders, step_scalars
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    s = UniPCMultistepScheduler(use_karras_sigmas=karras)
    s.set_timesteps(T)
    sig = torch.from_numpy(s.sigmas)
    p, c = orders(T)
    for i in range(T):
        k = step_scalars(sig, i, p[i], c[i])
        assert float(k["p_c"]) == float(k["p_aB"])                       # bh2: B_h = h_phi_1
        want = [k["sigma_s"], k["inv_alpha_s"], k["p_ratio"], k["p_c"], k.get("p_inv_rk", 0.0), p[i]]
        if c[i]:
            assert float(k["c_c"]) == float(k["c_aB"])
            rhos = [0.0, float(k["rhos_c"][0])] if c[i] == 1 else [float(v) for v in k["rhos_c"]]
            want += [k["c_ratio"], k["c_c"], k.get("c_inv_rk", 0.0)] + rhos + [c[i]]
        else:
            want += [0.0] * 6
        got = s.coeffs[i, :12].tolist()
        assert got == [float(v) for v in want], (i, got, want)
        assert s.coeffs[i, 12:].tolist() == [0.0] * 4 and np.isfinite(s.coeffs[i]).all()
        if c[i] == 2:
            assert s.coeffs[i, 9] != 0.0 and s.coeffs[i, 10] not in (0.0, 0.5)
    # the step to sigma 0: ratio 0 and c = -1, so the predictor returns x0 exactly
    assert s.coeffs[T - 1, 2] == 0.0 and s.coeffs[T - 1, 3] == -1.0


def test_from_config_and_refused_fields():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import EulerDiscreteScheduler, UniPCMultistepScheduler
    cfg = EulerDiscreteScheduler().config
    u = UniPCMultistepScheduler.from_config(cfg)
    assert isinstance(u, UniPCMultistepScheduler) and not u.use_karras_sigmas and u.kind == "unipc"
    k = UniPCMultistepScheduler.from_config(cfg, use_karras_sigmas=True)
    assert k.use_karras_sigmas and k.kind == "unipc_karras" and k.config["_class_name"] == "UniPCMultistepScheduler"
    with pytest.raises(TypeError):
        k.config["solver_order"] = 3                                    # read-only
    k.set_timesteps(20)
    assert k.timesteps[0] == 999
    again = UniPCMultistepScheduler.from_config(k.config, sample_max_value=2.0)
    again.set_timesteps(20)
    assert np.array_equal(again.coeffs, k.coeffs)
    for bad in (dict(solver_order=1), dict(solver_order=3), dict(solver_type="bh1"), dict(predict_x0=False),
                dict(disable_corrector=[0]), dict(solver_p=object()), dict(lower_order_final=False),
                dict(timestep_spacing="trailing"), dict(timestep_spacing="linspace"),
                dict(prediction_type="v_prediction"), dict(thresholding=True), dict(use_exponential_sigmas=True),
                dict(use_beta_sigmas=True), dict(rescale_betas_zero_snr=True), dict(final_sigmas_type="sigma_min"),
                dict(beta_schedule="linear"), dict(use_karas_sigmas=True)):
        with pytest.raises(IHError):
            UniPCMultistepScheduler.from_config(cfg, **bad)
    with pytest.raises(IHError):
        UniPCMultistepScheduler.from_config({**cfg, "timestep_spacing": "linspace"})


def test_from_config_moves_between_dpm_and_unipc_as_diffusers():
    """Euler -> DPM-Solver++ (Karras) -> UniPC -> DPM-Solver++ through `pipe.scheduler.config`, as a user swaps them:
    diffusers' constructors register UniPC's solver_type "bh2" for DPM-Solver's "midpoint" / "heun" / "logrho" and
    DPM-Solver++'s "midpoint" for "logrho" / "bh1" / "bh2", so each swap works and gives the scheduler built directly.
    Values that change the result stay refused: bh1 for UniPC, heun for DPM-Solver++, and unknown solver types."""
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, UniPCMultistepScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config, use_karras_sigmas=True)
    assert pipe.scheduler.config["solver_type"] == "midpoint"
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    uni = pipe.scheduler
    assert isinstance(uni, UniPCMultistepScheduler) and uni.kind == "unipc_karras"
    assert uni.config["solver_type"] == "bh2" and pipe.engine.scheduler is uni
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)
    dpm = pipe.scheduler
    assert isinstance(dpm, DPMSolverMultistepScheduler) and dpm.kind == "dpmpp_2m_karras"
    assert dpm.config["solver_type"] == "midpoint"
    for got, want in ((uni, UniPCMultistepScheduler(use_karras_sigmas=True)),
                      (dpm, DPMSolverMultistepScheduler(use_karras_sigmas=True))):
        assert dict(got.config) == dict(want.config)
        got.set_timesteps(10), want.set_timesteps(10)
        assert np.array_equal(got.timesteps, want.timesteps) and np.array_equal(got.coeffs, want.coeffs)
    for st in ("midpoint", "heun", "logrho", "bh2"):
        assert UniPCMultistepScheduler.from_config(dpm.config, solver_type=st).config["solver_type"] == "bh2"
    for st in ("midpoint", "logrho", "bh1", "bh2"):
        assert DPMSolverMultistepScheduler.from_config(uni.config, solver_type=st).config["solver_type"] == "midpoint"
    for bad in (lambda: UniPCMultistepScheduler.from_config(dpm.config, solver_type="bh1"),
                lambda: UniPCMultistepScheduler.from_config(dpm.config, solver_type="rk4"),
                lambda: DPMSolverMultistepScheduler.from_config(uni.config, solver_type="heun"),
                lambda: DPMSolverMultistepScheduler.from_config(uni.config, solver_type="rk4")):
        with pytest.raises(IHError):
            bad()


def _engine_vs_oracle(opts, karras, T=5, n=2, lat=8, seed=4, correct=True):
    from unipc_ref import UniPCRef, denoising_end_steps, unipc_denoise_loop
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    from oracle.scheduler_ref import prepare_latents
    native, ref = _build(TINY, seed)
    latents = prepare_latents(n, 4, lat, lat, [5, 6][:n], 1.0, dtype=torch.float32)
    _, ehs, te, tid = _inputs(TINY, n, lat, seed=9)
    procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    seen_ref, seen = [], []
    r = unipc_denoise_loop(lambda s, t, e, x, y: ref(s, t, e, x, y), latents.clone(), ehs[n:], ehs[:n], te[n:],
                           te[:n], tid[:n], T, karras=karras, set_scale=set_scale, conditioning_scale=0.8,
                           control_guidance_end=0.75, callback=lambda i, t, x: seen_ref.append((i, t, x.clone())),
                           callback_steps=2, correct=correct, **opts)
    eng = _fp32_engine(native)
    eng.scheduler = UniPCMultistepScheduler(use_karras_sigmas=karras)
    kw = dict(opts)
    loop_steps = denoising_end_steps(UniPCRef(T, karras).timesteps.tolist(), kw.pop("denoising_end", None))
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
def test_engine_matches_oracle_loop(unipc, opts, karras):
    """DenoiseEngine with UniPCMultistepScheduler on the stand-in ops vs unipc_denoise_loop: CFG and no CFG, rescale,
    denoising_end (its last step keeps predictor order 2), IP-scale gating and callback indices and timesteps."""
    o, r, seen, seen_ref, loop_steps = _engine_vs_oracle(opts, karras)
    if "denoising_end" in opts:
        assert 1 < loop_steps < 5
    assert torch.allclose(o, r, rtol=3e-4, atol=1e-3), (o - r).abs().max()
    assert [s[0] for s in seen] == [s[0] for s in seen_ref] == list(range(0, loop_steps, 2))
    assert [s[1] for s in seen] == [s[1] for s in seen_ref]
    for a, b in zip(seen, seen_ref):
        assert torch.allclose(a[2], b[2], rtol=3e-4, atol=1e-3)


def test_corrector_matters(unipc):
    """The corrector is really applied: the same loop without it (unipc_ref, correct=False) is more than 100 times
    further from the engine than the restatement with it."""
    o, r, *_ = _engine_vs_oracle(dict(guidance_scale=5.0), False)
    _, r_nc, *_ = _engine_vs_oracle(dict(guidance_scale=5.0), False, correct=False)
    assert (o - r_nc).abs().max() > 100 * (o - r).abs().max()


def test_engine_refuses_resume_and_image_options(unipc):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    native, _ = _build(TINY, 4)
    _, ehs, te, tid = _inputs(TINY, 1, 8)
    args = (torch.zeros(1, 4, 8, 8), ehs[1:], ehs[:1], te[1:], te[:1], tid[:1], 4)
    ip = (torch.zeros(1, 4, 8, 8), torch.zeros(1, 4, 8, 8), torch.ones(1, 1, 8, 8))
    cond = (torch.ones(1, 1, 8, 8), torch.zeros(1, 4, 8, 8))
    eng = _fp32_engine(native)
    eng.scheduler = UniPCMultistepScheduler()
    with _Empty32():
        for bad in (dict(begin_step=1), dict(inpaint=ip), dict(unet_cond=cond), dict(stop_after=2),
                    dict(start_step=1)):
            with pytest.raises(IHError, match="UniPCMultistepScheduler"):
                eng.run(*args, **bad)
        assert not eng._pool, "a refused call allocated a buffer"
        assert eng.run(*args).shape == (1, 4, 8, 8)


def test_text_to_image_pipeline_takes_a_unipc_scheduler(unipc):
    """scheduler= and `pipe.scheduler = ...` both work; the engine integrates that object; the initial latents are the
    plain noise (init_noise_sigma 1); denoising_end counts UniPC's timesteps."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerDiscreteScheduler, UniPCMultistepScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    emb = _embeds(1)
    common = dict(num_inference_steps=4, output_type="latent", height=64, width=64, **emb)
    uni = UniPCMultistepScheduler.from_config(EulerDiscreteScheduler().config, use_karras_sigmas=True)
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    pipe2 = StableDiffusionXLCustomPipeline(pipe.unet, scheduler=uni)
    assert pipe2.engine.scheduler is uni
    noise = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(2))
    assert torch.equal(pipe2.prepare_latents(1, 4, 64, 64, torch.float16, "cpu", torch.Generator().manual_seed(2)),
                       noise.half())
    calls = []
    a = pipe2(generator=torch.Generator().manual_seed(1), callback=lambda i, t, x: calls.append((i, int(t))),
              **common).images
    assert calls == [(i, int(t)) for i, t in enumerate(uni.timesteps)] and torch.isfinite(a.float()).all()
    e0 = pipe.engine
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    assert pipe.engine is not e0 and pipe.engine.scheduler is pipe.scheduler
    calls.clear()
    b = pipe(generator=torch.Generator().manual_seed(1), denoising_end=0.45,
             callback=lambda i, t, x: calls.append((i, int(t))), **common).images
    assert calls == [(0, 801), (1, 601)] and torch.isfinite(b.float()).all() and not torch.equal(a, b)


def test_img2img_and_inpaint_pipelines_refuse_unipc_before_any_work(unipc, monkeypatch):
    """Image-to-image (and so the refiner hand-over, which is an image-to-image call) and inpainting refuse UniPC
    before they encode a prompt or an image."""
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    pipe = _inpaint_pipe()
    pipe.scheduler = UniPCMultistepScheduler()

    def no_work(*a, **k):
        raise AssertionError("work was done before the scheduler was checked")
    monkeypatch.setattr(pipe.vae_encoder, "encode_moments_nhwc", no_work)
    monkeypatch.setattr(pipe, "encode_prompt", no_work)
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    common = dict(prompt="lions", num_inference_steps=4, output_type="latent", generator=torch.Generator().manual_seed(0))
    with pytest.raises(IHError, match="UniPCMultistepScheduler"):
        pipe(image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=0.5, height=64, width=64, **common)
    with pytest.raises(IHError, match="UniPCMultistepScheduler"):
        StableDiffusionXLImg2ImgPipeline.__call__(pipe, image=_pil_images(1)[0], strength=0.5, **common)
    with pytest.raises(IHError, match="UniPCMultistepScheduler"):
        StableDiffusionXLImg2ImgPipeline.__call__(pipe, image=torch.zeros(1, 4, 8, 8), strength=0.5,
                                                  denoising_start=0.8, **common)


def test_inpaint9_pipeline_refuses_unipc_before_any_work(monkeypatch):
    from test_inpaint9_cpu import _pipe9
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    pipe = _pipe9()
    pipe.scheduler = UniPCMultistepScheduler()

    def no_work(*a, **k):
        raise AssertionError("work was done before the scheduler was checked")
    monkeypatch.setattr(pipe, "encode_prompt", no_work)
    with pytest.raises(IHError, match="UniPCMultistepScheduler"):
        pipe(prompt="lions", image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=0.5, height=64, width=64,
             num_inference_steps=4, output_type="latent")


def test_ip_adapter_xl_generate_through_unipc_pipeline(unipc):
    """IPAdapterXL(pipe with a UniPC scheduler, ...).generate(...) with no change to ip_adapter.py."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import UniPCMultistepScheduler
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=[7, 8],
                  output_type="latent", height=64, width=64)
    euler = ip_model.generate(**common)
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config, use_karras_sigmas=True)
    a = ip_model.generate(**common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    assert (a.float() - euler.float()).abs().max() > 1e-2


def test_solver_step_entry_point_rejects_bad_arguments_before_any_launch():
    """ih_dpm_solver_step on the CPU-loaded library: UniPC without both extra history pointers, DPM-Solver++ with
    either of them, and an unknown solver are refused with an argument error before anything is launched."""
    from imagharmony_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(64)      # never dereferenced: the checks come first

    def call(solver, last_sample, prev_x0_2):
        return lib.ih_dpm_solver_step(p, p, p, p, p, p, p, 5.0, 0.0, 64, 1, 1, None, solver, last_sample, prev_x0_2)
    for solver, ls, p2 in ((_lib.IH_SOLVER_UNIPC_BH2, None, None), (_lib.IH_SOLVER_UNIPC_BH2, p, None),
                           (_lib.IH_SOLVER_UNIPC_BH2, None, p), (_lib.IH_SOLVER_DPMPP_2M, p, None),
                           (_lib.IH_SOLVER_DPMPP_2M, None, p), (_lib.IH_SOLVER_DPMPP_2M, p, p)):
        assert call(solver, ls, p2) == -1, (solver, ls, p2)
        assert b"last_sample and prev_x0_2" in lib.ih_last_error()
    for solver in (-1, 2, 7):
        assert call(solver, p, p) == -1 and b"solver" in lib.ih_last_error()
    # the shape and rescale checks still come before the launch with a valid solver
    assert lib.ih_dpm_solver_step(p, p, p, p, p, p, p, 5.0, 0.0, 1, 1, 1, None, 1, p, p) == -2
    assert lib.ih_dpm_solver_step(p, p, p, p, p, p, p, 5.0, 1.5, 64, 1, 1, None, 1, p, p) == -1
