"""CPU tests of image-to-image: the native VAE encoder's wiring, the folded conv_out / quant_conv, the scheduler's
strength truncation, DenoiseEngine.run(begin_step=...) and the StableDiffusionXLImg2ImgPipeline end to end, on the
plain-PyTorch stand-in ops (tests/fake_ops.py, tests/fake_ops_img2img.py) against the oracle (tests/img2img_ref.py)."""
import numpy as np
import pytest
import torch

import fake_ops_img2img
from test_wiring_cpu import _build, _Empty32, _fp32_engine, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def i2i(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_img2img.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_img2img, name))
    yield


def _encoder_pair(cfg, seed=0):
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(VAEEncoderRef(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, seed).items()}
    ref = VAEEncoderRef(cfg)
    ref.load_state_dict(sd)
    with torch.device("meta"):
        native = AutoencoderKLEncoder(cfg)
    native.load_state_dict(sd, assign=True)
    native.finalize()
    return native, ref.eval()


def _image(*shape, seed=0):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def test_vae_encoder_wiring_matches_oracle(i2i):
    from imagharmony_b200.config import TINY_VAE
    native, ref = _encoder_pair(TINY_VAE, seed=3)
    assert list(native.state_dict().keys()) == list(ref.state_dict().keys())      # diffusers key contract
    assert all(k.startswith(("encoder.", "quant_conv.")) for k in native.state_dict())
    x = _image(2, 3, 40, 56, seed=1)
    with torch.no_grad():
        r = ref.encode(x)
        o = native.encode(x)
    assert o.shape == r.shape == (2, 8, 5, 7)
    assert torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()


def test_vae_encoder_reads_a_full_vae_checkpoint(i2i):
    """from_state_dict takes the whole vae/diffusion_pytorch_model.safetensors dict (decoder keys present, ignored)."""
    from oracle.vae_ref import VAEDecoderRef
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.vae import AutoencoderKLDecoder, AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = {**shapes_of(VAEEncoderRef(TINY_VAE)), **shapes_of(VAEDecoderRef(TINY_VAE))}
    full = random_state_dict(shapes, 5)
    enc = AutoencoderKLEncoder.from_state_dict(TINY_VAE, full, device="cpu")
    dec = AutoencoderKLDecoder.from_state_dict(TINY_VAE, full, device="cpu")
    assert torch.equal(enc.quant_conv.weight, full["quant_conv.weight"]) and dec._w_in is not None
    with pytest.raises(KeyError):
        AutoencoderKLEncoder.from_state_dict(TINY_VAE, {k: v for k, v in full.items() if k != "quant_conv.bias"},
                                             device="cpu")


def test_vae_tiled_encode_matches_oracle(i2i):
    """enable_vae_tiling covers encode: an image larger than one 64-px tile (TINY_VAE) with ragged edge tiles is
    encoded tile-wise and its moments cross-faded like [3P] AutoencoderKL.tiled_encode; one tile takes the plain path."""
    from img2img_ref import tiled_encode_ref
    from imagharmony_b200.config import TINY_VAE
    native, ref = _encoder_pair(TINY_VAE, seed=4)
    native.use_tiling = True
    x = _image(1, 3, 104, 88, seed=2)                      # tiles at 0 / 48 / 96 rows, 0 / 48 columns
    with torch.no_grad():
        r = tiled_encode_ref(ref, x.clone())
        o = native.encode(x)
    assert o.shape == r.shape == (1, 8, 13, 11)
    assert torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()
    small = x[:, :, :64, :64].contiguous()
    with torch.no_grad():
        assert torch.allclose(native.encode(small), ref.encode(small), rtol=1e-4, atol=1e-4)


def test_vae_encoder_scaled_stream_is_exact_in_fp32(i2i):
    """The scaled residual stream of the encoder is the same function for k = 0, 7, 10, including a model whose
    stream exceeds 1e5 (beyond fp16 without the scaling)."""
    from imagharmony_b200.config import TINY_VAE
    native, ref = _encoder_pair(TINY_VAE, seed=5)
    assert native.stream_scale == 2.0 ** -7
    with torch.no_grad():
        for m in (native, ref):
            m.encoder.conv_in.weight.mul_(3e5)
            m.encoder.conv_in.bias.mul_(3e5)
    x = _image(1, 3, 24, 40, seed=3)
    with torch.no_grad():
        r = ref.encode(x)
        assert ref.encoder.conv_in(x).abs().max() > 1e5
    for k in (0, 7, 10):
        native.stream_scale = 2.0 ** -k
        native.finalize()
        with torch.no_grad():
            o = native.encode(x)
        assert torch.allclose(o, r, rtol=2e-4, atol=2e-4), (k, (o - r).abs().max())


def test_folded_conv_out_quant_conv_equals_two_convs():
    import torch.nn.functional as F
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        m = AutoencoderKLEncoder(TINY_VAE)
    m.load_state_dict({k: v.float() for k, v in random_state_dict(shapes_of(m), 6).items()}, assign=True)
    w, b = m.folded_conv_out()
    x = torch.randn(2, TINY_VAE.block_out_channels[-1], 5, 6, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        two = m.quant_conv(m.encoder.conv_out(x))
    one = F.conv2d(x, w, b, padding=1)
    assert torch.allclose(one, two, rtol=1e-5, atol=1e-5), (one - two).abs().max()


@pytest.mark.parametrize("T,strength,t_start", [(50, 0.3, 35), (30, 0.75, 8), (10, 1.0, 0), (4, 0.2, 4), (25, 0.5, 13),
                                                (10, 0.0, 10), (7, 0.99, 1)])
def test_scheduler_img2img_truncation(T, strength, t_start):
    from img2img_ref import img2img_timesteps
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from oracle.scheduler_ref import euler_tables
    s = EulerDiscreteScheduler()
    s.set_timesteps(T)
    assert s.img2img_begin_index(T, strength) == t_start
    rs, rts = img2img_timesteps(T, strength)
    assert rs == t_start and np.array_equal(s.timesteps[t_start:], rts)
    if t_start < T:
        assert s.add_noise_sigma(t_start) == float(euler_tables(T)[1][t_start])


@pytest.mark.parametrize("opts", [dict(), dict(denoising_end=0.6), dict(guidance_scale=1.0)])
def test_engine_begin_step_matches_oracle_loop(patched, opts):  # noqa: F811
    """DenoiseEngine.run(begin_step=t_start) vs the oracle loop over timesteps[t_start:]: sigma indices, IP-scale gating
    fractions and callback indices of the truncated list."""
    from img2img_ref import img2img_denoise_loop, img2img_timesteps
    from imagharmony_b200.config import TINY
    native, ref = _build(TINY, 4)
    T, strength, n, lat = 6, 0.7, 2, 8                        # t_start = 2, four steps
    t_start, ts = img2img_timesteps(T, strength)
    latents = torch.randn(n, 4, lat, lat, generator=torch.Generator().manual_seed(8)) * 3
    _, ehs, te, tid = _inputs(TINY, n, lat, seed=9)
    procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

    def set_scale(s):
        for p in procs:
            p.scale = s
    gs = opts.get("guidance_scale", 5.0)
    de = opts.get("denoising_end")
    seen_ref, seen = [], []
    r = img2img_denoise_loop(lambda s, t, e, x, y: ref(s, t, e, x, y), latents.clone(), ehs[n:], ehs[:n], te[n:], te[:n],
                             tid[:n], T, strength, guidance_scale=gs, set_scale=set_scale, conditioning_scale=0.8,
                             control_guidance_start=0.2, control_guidance_end=0.75, denoising_end=de,
                             callback=lambda i, t, x: seen_ref.append((i, float(t), x.clone())), callback_steps=2)
    loop_end = T
    if de is not None:
        loop_end = t_start + sum(1 for t in ts if t >= int(round(1000 - de * 1000)))
    eng = _fp32_engine(native)
    with _Empty32():
        o = eng.run(latents.clone(), ehs[n:], ehs[:n], te[n:], te[:n], tid[:n], T, guidance_scale=gs, ip_scale=0.8,
                    control_guidance_start=0.2, control_guidance_end=0.75, num_loop_steps=loop_end, begin_step=t_start,
                    callback=lambda i, t, x: seen.append((i, float(t), x.clone())), callback_steps=2)
    assert torch.allclose(o, r, rtol=3e-4, atol=1e-3), (o - r).abs().max()
    assert [s[:2] for s in seen] == [s[:2] for s in seen_ref] and seen[0][0] == 0
    for a, b in zip(seen, seen_ref):
        assert torch.allclose(a[2], b[2], rtol=3e-4, atol=1e-3)


def test_engine_begin_step_rejects_resume_options(patched):  # noqa: F811
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    native, _ = _build(TINY, 4)
    _, ehs, te, tid = _inputs(TINY, 1, 8)
    args = (torch.zeros(1, 4, 8, 8), ehs[1:], ehs[:1], te[1:], te[:1], tid[:1], 4)
    eng = _fp32_engine(native)
    with _Empty32():
        for bad in (dict(begin_step=1, start_step=2), dict(begin_step=1, stop_after=2), dict(begin_step=4),
                    dict(begin_step=2, num_loop_steps=2), dict(begin_step=-1)):
            with pytest.raises(IHError):
                eng.run(*args, **bad)


def _img2img_pipe():
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    pipe = StableDiffusionXLImg2ImgPipeline.from_random(TINY, seed=0, device="cpu", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict(random_state_dict(shapes_of(procs), 1))
    pipe.unet.finalize()
    return pipe


def _oracle_for(pipe):
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY, TINY_VAE
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    ref = UNetRef(TINY)
    procs = A.install_processors(ref, TINY)
    sd = {k: v.float() for k, v in pipe.unet.state_dict().items()}
    ref.load_state_dict(sd)
    venc = VAEEncoderRef(TINY_VAE)
    venc.load_state_dict({k: v.float() for k, v in pipe.vae_encoder.state_dict().items()})
    return ref.eval(), [p for p in procs.values() if hasattr(p, "to_k_ip")], venc.eval()


def _pil_images(n, size=(70, 64)):
    from PIL import Image
    rng = np.random.default_rng(0)
    return [Image.fromarray(rng.integers(0, 256, (size[1], size[0], 3), dtype=np.uint8)) for _ in range(n)]


@pytest.mark.parametrize("list_gen", [False, True])
def test_img2img_pipeline_matches_oracle(i2i, list_gen):
    """Two PIL images (70x64: floored to 64x64 and Lanczos-resized), a prompt batch of four: diffusers' RNG order
    (eps before noise, per generator) and its batch tiling (torch.cat of the encoded image batch), the noised start at
    sigma[t_start], the truncated loop with gating -- the pipeline on the stand-in ops vs the oracle chain."""
    from PIL import Image
    from img2img_ref import img2img_denoise_loop, img2img_timesteps, prepare_img2img_latents
    from imagharmony_b200.config import TINY, TINY_VAE
    from oracle.scheduler_ref import euler_tables
    pipe = _img2img_pipe()
    ref, procs, venc = _oracle_for(pipe)
    imgs = _pil_images(2)
    g = torch.Generator().manual_seed(11)
    pe, ne = torch.randn(4, 81, TINY.cross_attention_dim, generator=g).half(), torch.randn(4, 81, TINY.cross_attention_dim, generator=g).half()
    pp, npool = torch.randn(4, TINY.pooled_embed_dim, generator=g).half(), torch.randn(4, TINY.pooled_embed_dim, generator=g).half()
    T, strength = 5, 0.6

    def gens():
        return ([torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)] if list_gen
                else torch.Generator().manual_seed(1))
    pipe.set_scale(0.7)
    out = pipe(image=imgs, strength=strength, num_inference_steps=T, prompt_embeds=pe, negative_prompt_embeds=ne,
               pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npool, guidance_scale=5.0, generator=gens(),
               control_guidance_end=0.7, output_type="latent").images
    # oracle: VaeImageProcessor.preprocess -> prepare_latents -> loop
    pix = np.stack([np.array(im.resize((64, 64), resample=Image.LANCZOS)).astype(np.float32) / 255.0 for im in imgs])
    pix = torch.from_numpy(pix).permute(0, 3, 1, 2) * 2.0 - 1.0
    t_start, _ = img2img_timesteps(T, strength)
    sigma = float(euler_tables(T)[1][t_start])
    with torch.no_grad():
        lat = prepare_img2img_latents(venc.encode, pix, 4, gens(), sigma, TINY_VAE.scaling_factor)

    def set_scale(s):
        for p in procs:
            p.scale = s
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    r = img2img_denoise_loop(lambda s, t, e, x, y: ref(s.float(), t, e, x, y).half(), lat, pe.float(), ne.float(),
                             pp.float(), npool.float(), tid, T, strength, set_scale=set_scale, conditioning_scale=0.7,
                             control_guidance_end=0.7)
    err, mx = (out.float() - r.float()).abs().max().item(), r.float().abs().max().item()
    assert out.shape == (4, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    # the batch tiling is pinned: images in prompt order [0, 1, 0, 1] (torch.cat), not [0, 0, 1, 1]
    with torch.no_grad():
        swapped = prepare_img2img_latents(venc.encode, pix[[0, 0, 1, 1]] if list_gen else pix[[0, 1]], 4, gens(), sigma,
                                          TINY_VAE.scaling_factor)
    if not list_gen:
        swapped = swapped[[0, 2, 1, 3]]
    assert (swapped.float() - lat.float()).abs().max() > 0.1


def test_img2img_pipeline_arguments(i2i):
    from imagharmony_b200._lib import IHError
    pipe = _img2img_pipe()
    init = _image(1, 3, 64, 64, seed=4)
    common = dict(prompt="lions", num_inference_steps=4, output_type="latent", generator=torch.Generator().manual_seed(0))
    for bad in ("denoising_start", "timesteps", "sigmas", "latents"):
        with pytest.raises(IHError):
            pipe(image=init, strength=0.5, **{bad: 0.5 if bad == "denoising_start" else [1]}, **common)
    with pytest.raises(ValueError):                       # 4 * 0.2 -> no step left
        pipe(image=init, strength=0.2, **common)
    with pytest.raises(ValueError):
        pipe(image=init, strength=1.5, **common)
    with pytest.raises(ValueError):
        pipe(strength=0.5, **common)
    calls = []
    a = pipe(image=init, strength=0.5, number_class_crossattention=object(), aesthetic_score=9.0,
             negative_aesthetic_score=1.0, callback=lambda i, t, x: calls.append((i, int(t))), **common).images
    assert a.shape == (1, 4, 8, 8) and torch.isfinite(a.float()).all()
    assert calls == [(0, 251), (1, 1)]                       # timesteps[2:] of the 4-step schedule, indices from 0
    b = pipe(image=init, strength=0.5, denoising_end=0.8, **{**common, "generator": torch.Generator().manual_seed(0)}).images
    assert not torch.equal(a, b)                             # denoising_end keeps 1 of the 2 truncated steps
    # a [0, 1] tensor is normalised like VaeImageProcessor does; a [-1, 1] tensor is taken as it is
    from ip_adapter.custom_pipelines import preprocess_image
    x01 = (init + 1) / 2
    assert torch.allclose(preprocess_image(x01), init, atol=1e-6) and torch.equal(preprocess_image(init), init)
    assert preprocess_image(_pil_images(1, (21, 17))[0]).shape == (1, 3, 16, 16)


def test_ip_adapter_xl_generate_through_img2img_pipeline(i2i):
    """IPAdapterXL(img2img_pipe, ...).generate(pil_image=..., image=init, strength=s) with no change to ip_adapter.py."""
    from ip_adapter import IPAdapterXL
    pipe = _img2img_pipe()
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4, target_blocks=["down_blocks.2.attentions.1"],
                           inference=True)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    imgs = _pil_images(1)
    common = dict(clip_image_embeds=emb, prompt="lions", num_samples=2, num_inference_steps=4, seed=[7, 8],
                  output_type="latent")
    a = ip_model.generate(image=imgs[0], strength=0.5, **common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    b = ip_model.generate(image=imgs[0].transpose(0), strength=0.5, **common)      # another init image
    assert (a.float() - b.float()).abs().max() > 1e-2
    pil = ip_model.generate(image=imgs[0], strength=0.5, **{**common, "output_type": "pil"})
    assert len(pil) == 2 and pil[0].size == (64, 64)


def test_new_entry_points_reject_bad_arguments_before_any_launch():
    from imagharmony_b200 import _lib
    lib = _lib.load()
    # ih_conv2d_down_f16(x, w, bias, out, B, Hin, Win, Cin, Cout, tile_n, alpha, stream)
    assert lib.ih_conv2d_down_f16(None, 256, None, 256, 1, 16, 16, 64, 64, 0, 1.0, None) == -1
    assert b"null" in lib.ih_last_error()
    assert lib.ih_conv2d_down_f16(256, 256, None, 256, 1, 15, 16, 64, 64, 0, 1.0, None) == -2     # odd H
    assert lib.ih_conv2d_down_f16(256, 256, None, 256, 1, 16, 16, 60, 64, 0, 1.0, None) == -3     # Cin % 8
    # ih_vae_posterior_noise_f16(moments, ldc, eps, eps_f32, noise, out, B, Bm, Be, HW, C, sf, sigma, stream)
    assert lib.ih_vae_posterior_noise_f16(None, 16, 256, 1, 256, 256, 4, 2, 2, 64, 4, 0.13, 1.0, None) == -1
    assert lib.ih_vae_posterior_noise_f16(256, 16, 256, 1, 256, 256, 4, 3, 2, 64, 4, 0.13, 1.0, None) == -2   # B % Bm
    assert lib.ih_vae_posterior_noise_f16(256, 6, 256, 1, 256, 256, 4, 2, 2, 64, 4, 0.13, 1.0, None) == -2    # ldc < 2C
    assert lib.ih_vae_posterior_noise_f16(256, 16, 256, 2, 256, 256, 4, 2, 2, 64, 4, 0.13, 1.0, None) == -1   # eps_f32
