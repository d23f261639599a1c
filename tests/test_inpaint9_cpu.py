"""CPU tests of inpainting with the 9-channel inpainting UNet: the UNet's conv_in over latents | mask | masked-image
latents, DenoiseEngine.run(unet_cond=...), StableDiffusionXLInpaintPipeline end to end (Euler and Euler Ancestral)
with diffusers' RNG order, from_pretrained on a 9-channel checkpoint and the refusals -- on the plain-PyTorch
stand-in ops (tests/fake_ops*.py) against the oracle (tests/inpaint9_ref.py)."""
import dataclasses

import numpy as np
import pytest
import torch

import fake_ops_euler_a
import fake_ops_inpaint9
from test_img2img_cpu import _pil_images, i2i  # noqa: F401  (fixture)
from test_inpaint_cpu import _embeds, _pil_masks, inp  # noqa: F401  (fixture)
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def inp9(inp, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for mod in (fake_ops_inpaint9, fake_ops_euler_a):
        for name in mod.NAMES:
            monkeypatch.setattr(real_ops, name, getattr(mod, name))
    yield


def _tiny9():
    from imagharmony_b200.config import TINY
    return dataclasses.replace(TINY, in_channels=9)


def _pipe9():
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    pipe = StableDiffusionXLInpaintPipeline.from_random(_tiny9(), seed=0, device="cpu", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict(random_state_dict(shapes_of(procs), 1))
    pipe.unet.finalize()
    return pipe


def _oracle9_for(pipe):
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY_VAE
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    ref = UNetRef(_tiny9())
    procs = A.install_processors(ref, _tiny9())
    ref.load_state_dict({k: v.float() for k, v in pipe.unet.state_dict().items()})
    venc = VAEEncoderRef(TINY_VAE)
    venc.load_state_dict({k: v.float() for k, v in pipe.vae_encoder.state_dict().items()})
    return ref.eval(), [p for p in procs.values() if hasattr(p, "to_k_ip")], venc.eval()


def _pixels(imgs, size=64):
    from PIL import Image
    pix = np.stack([np.array(im.resize((size, size), resample=Image.LANCZOS)).astype(np.float32) / 255.0 for im in imgs])
    return torch.from_numpy(pix).permute(0, 3, 1, 2) * 2.0 - 1.0


def test_unet9_conv_in_wiring_matches_oracle(patched, monkeypatch):  # noqa: F811
    """The 9-channel UNet with `cond` (mask | masked latents read next to the latents) equals the oracle on the
    concatenated input; conv_in is packed to K = 128, the 4-channel one stays at K = 64."""
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    for name in fake_ops_inpaint9.NAMES:
        monkeypatch.setattr("imagharmony_b200.ops." + name, getattr(fake_ops_inpaint9, name))
    native, ref = _build(_tiny9(), 0)
    assert native._w_in.shape == (64, 128) and _build(TINY, 0)[0]._w_in.shape == (64, 64)
    sample, ehs, te, tid = _inputs(TINY, 1, 16)
    cond = torch.randn(2, 5, 16, 16, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        r = ref(torch.cat([sample, cond], 1), 321.0, ehs, te, tid)
        o = native(sample, torch.full((2,), 321.0), ehs, te, tid, cond=cond)
        assert o.shape == r.shape == (2, 4, 16, 16)
        assert torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()
        with pytest.raises(IHError):
            native(sample, torch.full((2,), 321.0), ehs, te, tid)                     # cond missing
        with pytest.raises(IHError):
            native(sample, torch.full((2,), 321.0), ehs, te, tid, cond=cond[:, :4])   # wrong shape
        four, _ = _build(TINY, 0)
        with pytest.raises(IHError):
            four(sample, torch.full((2,), 321.0), ehs, te, tid, cond=cond)            # the 4-channel UNet takes none


def test_unet_rejects_other_channel_counts(patched):  # noqa: F811
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    for c in (5, 8):
        with pytest.raises(IHError), torch.device("meta"):
            UNet2DConditionModel(dataclasses.replace(TINY, in_channels=c))
    with torch.device("meta"):
        shapes = shapes_of(UNet2DConditionModel(TINY))
    m = UNet2DConditionModel.from_state_dict(TINY, random_state_dict(shapes, 0), device="cpu")
    m.config = _tiny9()                              # a config that disagrees with conv_in.weight
    with pytest.raises(IHError):
        m.finalize()


def test_engine_unet_cond_matches_oracle_and_refuses(patched, monkeypatch):  # noqa: F811
    """run(unet_cond=(mask, masked)) vs the img2img oracle loop over the concatenated input, with begin_step, CFG,
    gating and callbacks; the argument checks."""
    from img2img_ref import img2img_denoise_loop, img2img_timesteps
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from inpaint9_ref import unet9_fn
    for name in fake_ops_inpaint9.NAMES:
        monkeypatch.setattr("imagharmony_b200.ops." + name, getattr(fake_ops_inpaint9, name))
    native, ref = _build(_tiny9(), 4)
    T, strength, n, lat = 6, 0.7, 2, 8
    t_start, _ = img2img_timesteps(T, strength)
    g = torch.Generator().manual_seed(8)
    latents = torch.randn(n, 4, lat, lat, generator=g) * 3
    mask = (torch.rand(n, 1, lat, lat, generator=g) > 0.5).float()
    masked = torch.randn(n, 4, lat, lat, generator=g)
    _, ehs, te, tid = _inputs(TINY, n, lat, seed=9)
    procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    seen_ref, seen = [], []
    r = img2img_denoise_loop(unet9_fn(lambda s, t, e, x, y: ref(s, t, e, x, y), mask, masked, True), latents.clone(),
                             ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], T, strength, set_scale=set_scale,
                             conditioning_scale=0.8, control_guidance_start=0.2,
                             callback=lambda i, t, x: seen_ref.append((i, float(t))))
    eng = _fp32_engine(native)
    args = (ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], T)
    with _Empty32():
        o = eng.run(latents.clone(), *args, ip_scale=0.8, control_guidance_start=0.2, begin_step=t_start,
                    unet_cond=(mask, masked), callback=lambda i, t, x: seen.append((i, float(t))))
        assert torch.allclose(o, r, rtol=3e-4, atol=1e-3), (o - r).abs().max()
        assert seen == seen_ref and seen[0][0] == 0
        ip = (torch.zeros(n, 4, lat, lat), torch.zeros(n, 4, lat, lat), torch.ones(n, 1, lat, lat))
        for bad in (dict(), dict(unet_cond=(mask, masked), inpaint=ip), dict(unet_cond=(mask, masked), start_step=1),
                    dict(unet_cond=(mask, masked), stop_after=2), dict(unet_cond=(mask[:1], masked)),
                    dict(unet_cond=(mask, masked[:, :3])), dict(unet_cond=(masked, mask))):
            with pytest.raises(IHError):
                eng.run(latents.clone(), *args, **bad)
        eng.scheduler = DPMSolverMultistepScheduler()
        with pytest.raises(IHError):
            eng.run(latents.clone(), *args, unet_cond=(mask, masked))
        four, _ = _build(TINY, 4)
        with pytest.raises(IHError):
            _fp32_engine(four).run(latents.clone(), *args, unet_cond=(mask, masked))


_CASES = [
    dict(strength=0.5, n_img=2, n_masks=1, list_gen=True),
    dict(strength=0.9999, n_img=1, n_masks=2, list_gen=False, guidance_rescale=0.7),
    dict(strength=1.0, n_img=2, n_masks=2, list_gen=False, guidance_scale=1.0),
    dict(strength=1.0, n_img=1, n_masks=1, list_gen=True, denoising_end=0.6, control_guidance_start=0.3),
    dict(strength=0.7, n_img=2, n_masks=1, list_gen=False, denoising_end=0.6),
    dict(strength=0.5, n_img=2, n_masks=1, list_gen=True, euler_a=True),
    dict(strength=1.0, n_img=1, n_masks=2, list_gen=False, euler_a=True, denoising_end=0.6),
    dict(strength=0.9999, n_img=1, n_masks=1, list_gen=False, euler_a=True, guidance_scale=1.0),
]


@pytest.mark.parametrize("opts", _CASES)
def test_inpaint9_pipeline_matches_oracle(inp9, opts):
    """Image(s) of 70x64 and mask(s) of 72x56 resized to 64x64, a prompt batch of four: start latents (no image encode
    at strength 1), mask and masked-image latents in diffusers' RNG order, the 9-channel model input, no blend; CFG /
    no CFG, rescale, denoising_end, gating, Euler and Euler A -- vs the oracle, and the generators end where the
    oracle's do."""
    from euler_a_ref import euler_a_denoise_loop
    from img2img_ref import img2img_denoise_loop, img2img_timesteps
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from inpaint_ref import preprocess_mask_ref
    from inpaint9_ref import prepare_inpaint9_inputs, unet9_fn
    opts = dict(opts)
    n_img, n_masks, list_gen = opts.pop("n_img"), opts.pop("n_masks"), opts.pop("list_gen")
    strength, euler_a = opts.pop("strength"), opts.pop("euler_a", False)
    pipe = _pipe9()
    if euler_a:
        pipe.scheduler = EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)
    ref, procs, venc = _oracle9_for(pipe)
    imgs, masks, emb = _pil_images(n_img), _pil_masks(n_masks), _embeds(4)
    T = 5

    def gens():
        return ([torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)] if list_gen
                else torch.Generator().manual_seed(1))
    pipe.set_scale(0.7)
    seen = []
    g_nat = gens()
    out = pipe(image=imgs if n_img > 1 else imgs[0], mask_image=masks if n_masks > 1 else masks[0], strength=strength,
               num_inference_steps=T, height=64, width=64, generator=g_nat, control_guidance_end=0.8,
               output_type="latent", callback=lambda i, t, x: seen.append((i, int(t))), **opts, **emb).images
    t_start, ts = img2img_timesteps(T, strength)
    g_ref = gens()
    mask = preprocess_mask_ref(masks, 64, 64)
    with torch.no_grad():
        lat, m, ml = prepare_inpaint9_inputs(venc.encode, _pixels(imgs), mask, 4, g_ref, t_start, T, strength,
                                             TINY_VAE.scaling_factor)

    def set_scale(s):
        for p in procs:
            p.scale = s
    gs = opts.pop("guidance_scale", 7.5)
    fn = unet9_fn(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), m, ml, gs > 1.0)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    embf = [emb[k].float() for k in ("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                                     "negative_pooled_prompt_embeds")]
    seen_ref = []
    common = dict(guidance_scale=gs, set_scale=set_scale, conditioning_scale=0.7, control_guidance_end=0.8,
                  callback=lambda i, t, x: seen_ref.append((i, int(t))), **opts)
    if euler_a:
        r = euler_a_denoise_loop(fn, lat, *embf, tid, T, generator=g_ref, begin=t_start, **common)
    else:
        r = img2img_denoise_loop(fn, lat, *embf, tid, T, strength, **common)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (4, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    assert seen == seen_ref and len(seen) >= 1 and seen[0] == (0, int(ts[0]))
    for a, b in zip(g_nat if list_gen else [g_nat], g_ref if list_gen else [g_ref]):
        assert torch.equal(a.get_state(), b.get_state())


@pytest.mark.parametrize("strength", [0.5, 1.0])
@pytest.mark.parametrize("list_gen", [False, True])
def test_generator_consumption_order(inp9, strength, list_gen):
    """One generator: [eps of the image batch (strength < 1)] -> noise of the whole batch -> eps of the masked images.
    A list: the same per generator, image / masked image i drawing with generator[i] (SURVEY C.32)."""
    pipe = _pipe9()
    emb = _embeds(3)
    seeds = (5, 6, 7)
    gens = [torch.Generator().manual_seed(s) for s in seeds] if list_gen else torch.Generator().manual_seed(5)
    pipe(image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=strength, num_inference_steps=4, height=64,
         width=64, generator=gens, output_type="latent", **emb)
    if list_gen:
        want = [torch.Generator().manual_seed(s) for s in seeds]
        if strength < 1:
            torch.randn((1, 4, 8, 8), generator=want[0], dtype=torch.float32)
        for w in want:
            torch.randn((1, 4, 8, 8), generator=w, dtype=torch.float16)
        torch.randn((1, 4, 8, 8), generator=want[0], dtype=torch.float32)
        assert all(torch.equal(a.get_state(), b.get_state()) for a, b in zip(gens, want))
    else:
        want = torch.Generator().manual_seed(5)
        if strength < 1:
            torch.randn((1, 4, 8, 8), generator=want, dtype=torch.float32)
        torch.randn((3, 4, 8, 8), generator=want, dtype=torch.float16)
        torch.randn((1, 4, 8, 8), generator=want, dtype=torch.float32)
        assert torch.equal(gens.get_state(), want.get_state())


def test_inpaint9_pipeline_arguments(inp9):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline, StableDiffusionXLImg2ImgPipeline
    pipe = _pipe9()
    img, mask = _pil_images(1)[0], _pil_masks(1)[0]
    common = dict(prompt="lions", num_inference_steps=4, output_type="latent", height=64, width=64,
                  generator=torch.Generator().manual_seed(0))
    for bad in ("masked_image_latents", "padding_mask_crop", "denoising_start"):
        with pytest.raises(IHError):
            pipe(image=img, mask_image=mask, strength=0.5, **{bad: 32 if bad == "padding_mask_crop" else [1]}, **common)
    with pytest.raises(ValueError):                                   # 2 images and 3 masks do not broadcast
        pipe(image=_pil_images(2), mask_image=_pil_masks(3), strength=0.5, num_images_per_prompt=6, **common)
    with pytest.raises(ValueError):                                   # 3 masks do not divide a batch of 2
        pipe(image=img, mask_image=_pil_masks(3), strength=0.5, num_images_per_prompt=2, **common)
    with pytest.raises(ValueError):
        pipe(image=img, mask_image=mask, strength=0.5,
             **{**common, "generator": [torch.Generator().manual_seed(0)] * 2})
    a = pipe(image=img, mask_image=mask, strength=0.5, **common).images
    assert a.shape == (1, 4, 8, 8) and torch.isfinite(a.float()).all()
    # text-to-image and image-to-image have no mask to feed a 9-channel UNet
    with pytest.raises(IHError):
        StableDiffusionXLCustomPipeline(pipe.unet)(prompt="lions", num_inference_steps=2, height=64, width=64,
                                                   output_type="latent")
    with pytest.raises(IHError):
        StableDiffusionXLImg2ImgPipeline(pipe.unet, vae_encoder=pipe.vae_encoder)(
            prompt="lions", image=img, strength=0.5, num_inference_steps=4, output_type="latent")
    pipe.scheduler = DPMSolverMultistepScheduler()
    with pytest.raises(IHError):
        pipe(image=img, mask_image=mask, strength=0.5, **common)


def test_from_pretrained_reads_the_channel_count_of_the_checkpoint(inp9, tmp_path, monkeypatch):
    """Without `cfg`, from_pretrained builds the UNet with the input channels of the checkpoint's conv_in: a 9-channel
    snapshot loads as the inpainting UNet and runs the 9-channel path, a 4-channel one keeps the default config."""
    from safetensors.torch import save_file
    import ip_adapter.custom_pipelines as cp
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    monkeypatch.setattr(cp, "SDXL_BASE", TINY)                  # the default architecture, at test size
    for c, sub in ((9, "inpaint"), (4, "base")):
        root = tmp_path / sub
        for d in ("unet", "vae"):
            (root / d).mkdir(parents=True)
        with torch.device("meta"):
            ushapes = shapes_of(UNet2DConditionModel(dataclasses.replace(TINY, in_channels=c)))
            vshapes = {**shapes_of(AutoencoderKLDecoder(TINY_VAE)), **shapes_of(VAEEncoderRef(TINY_VAE))}
        usd = random_state_dict(ushapes, 1)
        save_file({k: v.contiguous() for k, v in usd.items()}, str(root / "unet" / "diffusion_pytorch_model.safetensors"))
        save_file({k: v.contiguous() for k, v in random_state_dict(vshapes, 2).items()},
                  str(root / "vae" / "diffusion_pytorch_model.safetensors"))
        pipe = cp.StableDiffusionXLInpaintPipeline.from_pretrained(str(root), device="cpu", vae_cfg=TINY_VAE)
        assert pipe.unet.config.in_channels == c and pipe.unet.conv_in.weight.shape[1] == c
        assert torch.equal(pipe.unet.conv_in.weight, usd["conv_in.weight"])
        if c == 4:
            assert pipe.unet.config is TINY
        calls = []
        run = pipe.engine.run
        pipe.engine.run = lambda *a, **k: calls.append(k["unet_cond"] is not None) or run(*a, **k)
        out = pipe(prompt="lions", image=_pil_images(1)[0], mask_image=_pil_masks(1)[0], strength=0.5,
                   num_inference_steps=4, height=64, width=64, generator=torch.Generator().manual_seed(0),
                   output_type="latent").images
        assert out.shape == (1, 4, 8, 8) and torch.isfinite(out.float()).all() and calls == [c == 9]


def test_ip_adapter_xl_generate_through_inpaint9_pipeline(inp9):
    """IPAdapterXL(pipe with the 9-channel UNet, ...).generate(pil_image=..., image=init, mask_image=mask) with no
    change to ip_adapter.py; the mask reaches the UNet (another mask, another result)."""
    from PIL import Image
    from ip_adapter import IPAdapterXL
    pipe = _pipe9()
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    img, mask = _pil_images(1)[0], _pil_masks(1)[0]
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=[7, 8],
                  output_type="latent", height=64, width=64)
    a = ip_model.generate(image=img, mask_image=mask, strength=1.0, **common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    b = ip_model.generate(image=img, mask_image=Image.new("L", mask.size, 255), strength=1.0, **common)
    assert (a.float() - b.float()).abs().max() > 1e-2
    pil = ip_model.generate(image=img, mask_image=mask, strength=0.7, **{**common, "output_type": "pil"})
    assert len(pil) == 2 and pil[0].size == (64, 64)


def test_im2col_cat_rejects_bad_arguments_before_any_launch():
    from imagharmony_b200 import _lib
    lib = _lib.load()
    # ih_im2col3x3_nchw_cat_f16(x0, C0, x1, C1, out, B, H, W, Kpad, stream)
    assert lib.ih_im2col3x3_nchw_cat_f16(None, 4, 256, 5, 256, 1, 8, 8, 128, None) == -1
    assert lib.ih_im2col3x3_nchw_cat_f16(256, 4, None, 5, 256, 1, 8, 8, 128, None) == -1
    assert lib.ih_im2col3x3_nchw_cat_f16(256, 4, 256, 5, 256, 1, 8, 8, 84, None) == -1     # Kpad % 8
    assert lib.ih_im2col3x3_nchw_cat_f16(256, 4, 256, 5, 256, 1, 8, 8, 80, None) == -1     # Kpad < 81
    assert lib.ih_im2col3x3_nchw_cat_f16(256, 4, 256, 0, 256, 1, 8, 8, 128, None) == -2     # empty
