"""CPU tests of inpainting with the 4-channel UNet: mask preprocessing, DenoiseEngine.run(inpaint=...) and the
StableDiffusionXLInpaintPipeline end to end on the plain-PyTorch stand-in ops (tests/fake_ops.py,
tests/fake_ops_img2img.py, tests/fake_ops_inpaint.py) against the oracle (tests/inpaint_ref.py)."""
import dataclasses

import numpy as np
import pytest
import torch

import fake_ops_inpaint
from test_img2img_cpu import _oracle_for, _pil_images, i2i  # noqa: F401  (fixture)
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def inp(i2i, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_inpaint.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_inpaint, name))
    yield


def _inpaint_pipe():
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    pipe = StableDiffusionXLInpaintPipeline.from_random(TINY, seed=0, device="cpu", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict(random_state_dict(shapes_of(procs), 1))
    pipe.unet.finalize()
    return pipe


def _pil_masks(n, size=(72, 56)):
    """Masks with a regenerated rectangle (255), a kept border (0) and values around 0.5 at a seam."""
    from PIL import Image
    out = []
    for k in range(n):
        a = np.zeros((size[1], size[0]), dtype=np.uint8)
        a[8 + 4 * k:40, 16:60 - 8 * k] = 255
        a[44:48, :] = 127 + k          # 127/255 < 0.5 <= 128/255
        out.append(Image.fromarray(a).convert("RGB"))
    return out


def _embeds(n, seed=11):
    from imagharmony_b200.config import TINY
    g = torch.Generator().manual_seed(seed)
    pe, ne = (torch.randn(n, 81, TINY.cross_attention_dim, generator=g).half() for _ in range(2))
    pp, npool = (torch.randn(n, TINY.pooled_embed_dim, generator=g).half() for _ in range(2))
    return dict(prompt_embeds=pe, negative_prompt_embeds=ne, pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npool)


@pytest.mark.parametrize("opts", [
    dict(strength=0.5, n_img=2, n_masks=1, list_gen=True),
    dict(strength=0.5, n_img=1, n_masks=2, list_gen=False, guidance_rescale=0.7),
    dict(strength=1.0, n_img=2, n_masks=1, list_gen=True),
    dict(strength=1.0, n_img=2, n_masks=2, list_gen=False, guidance_scale=1.0),
    dict(strength=0.9999, n_img=1, n_masks=1, list_gen=False, denoising_end=0.6),
    dict(strength=0.7, n_img=2, n_masks=1, list_gen=False, denoising_end=0.6, control_guidance_start=0.3),
])
def test_inpaint_pipeline_matches_oracle(inp, opts):
    """Image(s) of 70x64 and mask(s) of 72x56 resized to the requested 64x64, a prompt batch of four: image latents,
    noise and start latents in diffusers' RNG order, mask latents, the blend after every step (the last one with the
    clean latents, also when denoising_end stops early), CFG / no CFG, rescale, gating -- on the stand-in ops vs the
    oracle chain."""
    from PIL import Image
    from img2img_ref import img2img_timesteps
    from imagharmony_b200.config import TINY_VAE
    from inpaint_ref import inpaint_denoise_loop, mask_latents_ref, prepare_inpaint_latents, preprocess_mask_ref
    opts = dict(opts)
    n_img, n_masks, list_gen = opts.pop("n_img"), opts.pop("n_masks"), opts.pop("list_gen")
    strength = opts.pop("strength")
    pipe = _inpaint_pipe()
    ref, procs, venc = _oracle_for(pipe)
    imgs, masks = _pil_images(n_img), _pil_masks(n_masks)
    emb = _embeds(4)
    T = 5

    def gens():
        return ([torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)] if list_gen
                else torch.Generator().manual_seed(1))
    pipe.set_scale(0.7)
    seen = []
    out = pipe(image=imgs if n_img > 1 else imgs[0], mask_image=masks if n_masks > 1 else masks[0], strength=strength,
               num_inference_steps=T, height=64, width=64, generator=gens(), control_guidance_end=0.8,
               output_type="latent", callback=lambda i, t, x: seen.append((i, int(t))), **opts, **emb).images
    pix = np.stack([np.array(im.resize((64, 64), resample=Image.LANCZOS)).astype(np.float32) / 255.0 for im in imgs])
    pix = torch.from_numpy(pix).permute(0, 3, 1, 2) * 2.0 - 1.0
    t_start, ts = img2img_timesteps(T, strength)
    with torch.no_grad():
        lat, img_lat, noise = prepare_inpaint_latents(venc.encode, pix, 4, gens(), t_start, T, strength,
                                                      TINY_VAE.scaling_factor)
    mask = mask_latents_ref(preprocess_mask_ref(masks, 64, 64), 4, 64, 64)

    def set_scale(s):
        for p in procs:
            p.scale = s
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    seen_ref = []
    r = inpaint_denoise_loop(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), lat, img_lat, noise, mask,
                             emb["prompt_embeds"].float(), emb["negative_prompt_embeds"].float(),
                             emb["pooled_prompt_embeds"].float(), emb["negative_pooled_prompt_embeds"].float(), tid, T,
                             strength, set_scale=set_scale, conditioning_scale=0.7, control_guidance_end=0.8,
                             callback=lambda i, t, x: seen_ref.append((i, int(t))), **opts)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (4, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    assert seen == seen_ref and len(seen) >= 1 and seen[0] == (0, int(ts[0]))
    # outside the mask the result is the clean image latents (up to the fp32 oracle's encoder), inside it is not
    keep = (mask == 0).expand_as(r)
    assert (out.float() - img_lat.float())[keep].abs().max() <= 2e-2 * mx
    assert (out.float() - img_lat.float())[~keep].abs().max() > 0.1


@pytest.mark.parametrize("T", [30, 50])
def test_default_strength_skips_the_first_step(T):
    from img2img_ref import img2img_timesteps
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    s = EulerDiscreteScheduler()
    s.set_timesteps(T)
    assert s.img2img_begin_index(T, 0.9999) == 1 == img2img_timesteps(T, 0.9999)[0]


def test_inpaint_pipeline_defaults(inp):
    """strength 0.9999 (T = 30: 29 steps from timesteps[1]), guidance_scale 7.5 (CFG on), height / width from the UNet's
    sample size, not from the image's size."""
    import inspect
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    sig = inspect.signature(StableDiffusionXLInpaintPipeline.__call__).parameters
    assert sig["strength"].default == 0.9999 and sig["guidance_scale"].default == 7.5
    assert sig["height"].default is None and sig["width"].default is None
    pipe = _inpaint_pipe()
    calls = []
    pipe.engine.run_orig = pipe.engine.run

    def spy(*a, **k):
        calls.append((a[0].shape, k["guidance_scale"], k["begin_step"]))
        return pipe.engine.run_orig(*a, **k)
    pipe.engine.run = spy
    seen = []
    out = pipe(prompt="lions", image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], num_inference_steps=30,
               generator=torch.Generator().manual_seed(0), output_type="latent",
               callback=lambda i, t, x: seen.append(int(t))).images
    size = pipe.default_sample_size
    assert out.shape == (1, 4, size, size) and calls == [((1, 4, size, size), 7.5, 1)]
    assert len(seen) == 29 and seen[0] == int(pipe.scheduler.timesteps[1])


def test_preprocess_mask_matches_oracle():
    from PIL import Image
    from inpaint_ref import preprocess_mask_ref
    from ip_adapter.custom_pipelines import preprocess_mask
    rgb = _pil_masks(2)
    rgba = [m.convert("RGBA") for m in rgb]
    gray = [m.convert("L") for m in rgb]
    for m in (rgb[0], rgba, gray, gray[1]):
        for hw in ((56, 72), (64, 64), (40, 96)):
            a, b = preprocess_mask(m, *hw), preprocess_mask_ref(m, *hw)
            assert a.shape == b.shape == (len(m) if isinstance(m, list) else 1, 1) + hw and torch.equal(a, b)
    # the 0.5 threshold on exact values: 127 -> 0, 128 -> 1 (no resize)
    seam = Image.fromarray(np.array([[127, 128] * 4] * 8, dtype=np.uint8))
    assert preprocess_mask(seam, 8, 8)[0, 0, 0].tolist() == [0.0, 1.0] * 4
    g = torch.Generator().manual_seed(3)
    for t in (torch.rand(2, 1, 24, 40, generator=g), torch.rand(3, 24, 40, generator=g), torch.rand(24, 40, generator=g)):
        a, b = preprocess_mask(t, 48, 32), preprocess_mask_ref(t, 48, 32)
        assert a.shape == b.shape and a.shape[1:] == (1, 48, 32) and torch.equal(a, b)
        assert set(a.unique().tolist()) <= {0.0, 1.0}
    with pytest.raises(ValueError):
        preprocess_mask(torch.rand(2, 3, 8, 8), 8, 8)


def test_mask_latents_read_one_pixel_per_block():
    """diffusers' nearest interpolate to the latent size reads mask[..., ::8, ::8] (SURVEY C.20)."""
    from inpaint_ref import mask_latents_ref
    m = (torch.rand(2, 1, 64, 48, generator=torch.Generator().manual_seed(4)) > 0.5).float()
    lat = mask_latents_ref(m, 4, 64, 48)
    assert lat.dtype == torch.float16 and torch.equal(lat, m[..., ::8, ::8].half().repeat(2, 1, 1, 1))
    with pytest.raises(ValueError):
        mask_latents_ref(m, 3, 64, 48)


@pytest.mark.parametrize("list_gen", [False, True])
def test_generator_consumption_order(inp, list_gen):
    """One generator: eps for the image batch, then the noise of the whole batch.  A list: generator[i] draws eps for
    image i < n_images, then every generator draws its slot's noise (SURVEY C.19)."""
    pipe = _inpaint_pipe()
    emb = _embeds(3)
    gens = [torch.Generator().manual_seed(s) for s in (5, 6, 7)] if list_gen else torch.Generator().manual_seed(5)
    pipe(image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=0.5, num_inference_steps=4, height=64, width=64,
         generator=gens, output_type="latent", **emb)
    if list_gen:
        want = [torch.Generator().manual_seed(s) for s in (5, 6, 7)]
        torch.randn((1, 4, 8, 8), generator=want[0], dtype=torch.float32)
        for w in want:
            torch.randn((1, 4, 8, 8), generator=w, dtype=torch.float16)
        assert all(torch.equal(a.get_state(), b.get_state()) for a, b in zip(gens, want))
    else:
        want = torch.Generator().manual_seed(5)
        torch.randn((1, 4, 8, 8), generator=want, dtype=torch.float32)
        torch.randn((3, 4, 8, 8), generator=want, dtype=torch.float16)
        assert torch.equal(gens.get_state(), want.get_state())


def test_inpaint_pipeline_arguments(inp, monkeypatch):
    from imagharmony_b200._lib import IHError
    pipe = _inpaint_pipe()
    img, mask = _pil_images(1)[0], _pil_masks(1)[0]
    common = dict(prompt="lions", num_inference_steps=4, output_type="latent", height=64, width=64,
                  generator=torch.Generator().manual_seed(0))
    for bad in ("denoising_start", "timesteps", "sigmas", "latents", "ip_adapter_image", "ip_adapter_image_embeds",
                "clip_skip", "callback_on_step_end", "masked_image_latents", "padding_mask_crop"):
        with pytest.raises(IHError):
            pipe(image=img, mask_image=mask, strength=0.5, **{bad: 32 if bad == "padding_mask_crop" else [1]}, **common)
    for bad in (dict(strength=1.5), dict(strength=-0.1), dict(height=60), dict(width=100), dict(strength=0.2),
                dict(mask_image=None), dict(image=None)):
        with pytest.raises(ValueError):
            pipe(**{"image": img, "mask_image": mask, "strength": 0.5, **common, **bad})
    with pytest.raises(ValueError):                                   # 3 masks do not divide a batch of 2
        pipe(image=img, mask_image=_pil_masks(3), strength=0.5, num_images_per_prompt=2,
             **{k: v for k, v in common.items() if k != "prompt"}, prompt="lions")
    a = pipe(image=img, mask_image=mask, strength=0.5, number_class_crossattention=object(), aesthetic_score=9.0,
             negative_aesthetic_score=1.0, **common).images
    assert a.shape == (1, 4, 8, 8) and torch.isfinite(a.float()).all()
    monkeypatch.setattr(pipe.unet, "config", dataclasses.replace(pipe.unet.config, in_channels=9))
    with pytest.raises(IHError):
        pipe(image=img, mask_image=mask, strength=0.5, **common)


def test_engine_inpaint_rejects_resume_options(patched):  # noqa: F811
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    native, _ = _build(TINY, 4)
    _, ehs, te, tid = _inputs(TINY, 1, 8)
    args = (torch.zeros(1, 4, 8, 8), ehs[1:], ehs[:1], te[1:], te[:1], tid[:1], 4)
    ip = (torch.zeros(1, 4, 8, 8), torch.zeros(1, 4, 8, 8), torch.ones(1, 1, 8, 8))
    eng = _fp32_engine(native)
    with _Empty32():
        for bad in (dict(start_step=1), dict(stop_after=2), dict(begin_step=1, stop_after=2)):
            with pytest.raises(IHError):
                eng.run(*args, inpaint=ip, **bad)
        with pytest.raises(IHError):
            eng.run(*args, inpaint=(ip[0], ip[1], torch.ones(1, 4, 8, 8)))


def test_ip_adapter_xl_generate_through_inpaint_pipeline(inp):
    """IPAdapterXL(inpaint_pipe, ...).generate(pil_image=..., image=init, mask_image=mask, strength=s) with no change
    to ip_adapter.py."""
    from ip_adapter import IPAdapterXL
    pipe = _inpaint_pipe()
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    img, mask = _pil_images(1)[0], _pil_masks(1)[0]
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=[7, 8],
                  output_type="latent", height=64, width=64)
    a = ip_model.generate(image=img, mask_image=mask, strength=0.7, **common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    from PIL import Image
    b = ip_model.generate(image=img, mask_image=Image.new("L", mask.size, 255), strength=0.7, **common)  # regenerate all
    assert (a.float() - b.float()).abs().max() > 1e-2
    pil = ip_model.generate(image=img, mask_image=mask, strength=0.7, **{**common, "output_type": "pil"})
    assert len(pil) == 2 and pil[0].size == (64, 64)
