"""GPU tests of inpainting with the 4-channel UNet: the fused Euler + mask-blend step kernel against a torch restatement
of its rounding points (tests/inpaint_ref.py), the graph-replayed pipeline against the fp32 oracle trajectory, the
bit-exact invariants that tie it to the clean image, to text-to-image and to image-to-image, and graph reuse when the
three run alternately on one engine."""
import numpy as np
import pytest
import torch

from test_img2img_gpu import _pipe_and_oracles
from test_kernels_gpu import STEP_BUCKETS, check, ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("frac", [False, True])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("use_cfg,rescale,hw", [
    pytest.param(True, 0.0, (64, 48), id="True-0.0"), pytest.param(False, 0.0, (64, 48), id="False-0.0"),
    pytest.param(True, 0.7, (64, 48), id="True-0.7"),
] + [pytest.param(True, 0.7, hw, id=f"True-0.7-{hw[0]}x{hw[1]}") for hw in STEP_BUCKETS])
def test_euler_inpaint_step_kernel(ops, use_cfg, rescale, n, frac, hw):  # noqa: F811
    """Steps at the start, in the middle, at blend_end - 1 (the last step of a denoising_end loop: blends with the clean
    latents although sigma[i+1] > 0) and at the end of a 10-step schedule.  Without rescale bit-exact (no fast math:
    IEEE division and sqrt; FMA contraction restated); with rescale the bar of test_kernels_gpu.py::test_euler_step_ex,
    since the per-image std is a reduction in another order than torch's."""
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from inpaint_ref import inpaint_step_ref
    T, (h, w) = 10, hw
    sig_np = EulerDiscreteScheduler().set_timesteps(T).sigmas
    sig = torch.from_numpy(sig_np).cuda()
    b = 2 * n if use_cfg else n
    g = torch.Generator().manual_seed(100 * n + 10 * int(use_cfg) + int(frac))
    for i, end in ((0, 10), (4, 10), (6, 7), (9, 10)):
        lat = (torch.randn(n, 4, h, w, generator=g) * float(sig_np[i])).half().cuda()
        noise_pred = torch.randn(b, 4, h, w, generator=g).half().cuda()
        img = torch.randn(n, 4, h, w, generator=g).half().cuda()
        nz = torch.randn(n, 4, h, w, generator=g).half().cuda()
        m = torch.rand(n, 1, h, w, generator=g)
        m = (m if frac else (m > 0.5).float()).half().cuda()
        ref_x, ref_mi = inpaint_step_ref(noise_pred, lat, sig_np, i, 7.5, img, nz, m, end, use_cfg, rescale)
        step = torch.tensor([i], dtype=torch.int32, device="cuda")
        blend_end = torch.tensor([end], dtype=torch.int32, device="cuda")
        model_in = torch.empty(b, 4, h, w, dtype=torch.float16, device="cuda")
        ops.euler_inpaint_step(noise_pred, lat, model_in, sig, step, 7.5, img, nz, m, blend_end, use_cfg=use_cfg,
                               guidance_rescale=rescale)
        assert int(step.item()) == i + 1
        what = f"euler_inpaint cfg={use_cfg} r={rescale} n={n} frac={frac} step {i} end {end}"
        if rescale == 0.0:
            exact = (lat == ref_x).float().mean().item()
            print(f"[{what}] bit-exact latents {exact:.6f}")
            assert torch.equal(lat, ref_x) and torch.equal(model_in, ref_mi), what
        else:
            check(lat, ref_x, what, rtol=2e-3, atol=2e-3)
            check(model_in, ref_mi, what + " model_in", rtol=2e-3, atol=2e-3)


@pytest.fixture(scope="module")
def pipes():
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    i2i, oracles = _pipe_and_oracles()
    inp = StableDiffusionXLInpaintPipeline(i2i.unet, vae=i2i.vae, vae_encoder=i2i.vae_encoder)
    return i2i, inp, oracles


def _images(n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    return [Image.fromarray(rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)) for _ in range(n)]


def _mask(value=None):
    from PIL import Image
    if value is not None:
        return Image.new("L", (64, 64), value)
    a = np.zeros((64, 64), dtype=np.uint8)
    a[8:40, 16:56] = 255
    return Image.fromarray(a)


def _emb(batch=4):
    from imagharmony_b200.config import TINY
    g = torch.Generator().manual_seed(11)
    pe, ne = (torch.randn(batch, 81, TINY.cross_attention_dim, generator=g).half() for _ in range(2))
    pp, npool = (torch.randn(batch, TINY.pooled_embed_dim, generator=g).half() for _ in range(2))
    return dict(prompt_embeds=pe, negative_prompt_embeds=ne, pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npool)


def _gens():
    return [torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)]


def test_inpaint_graph_replayed_matches_oracle_trajectory(pipes):
    """TINY UNet + TINY_VAE, CFG 7.5, IP scale 0.7 gated off for the last step, strength 0.5 of 6 steps, two images and
    one mask tiled to a prompt batch of four, a list of generators, graph-replayed -- vs the fp32 oracle trajectory with
    the bar of SURVEY section 7."""
    from imagharmony_b200.config import TINY_VAE
    from img2img_ref import img2img_timesteps
    from inpaint_ref import inpaint_denoise_loop, mask_latents_ref, prepare_inpaint_latents, preprocess_mask_ref
    _, pipe, oracles = pipes
    imgs, mask, emb = _images(2), _mask(), _emb()
    T, strength = 6, 0.5
    pipe.set_scale(0.7)
    o = pipe(image=imgs, mask_image=mask, strength=strength, num_inference_steps=T, height=64, width=64,
             generator=_gens(), control_guidance_end=0.7, output_type="latent", **emb).images
    torch.cuda.synchronize()
    pix = torch.from_numpy(np.stack([np.array(im).astype(np.float32) / 255.0 for im in imgs])).permute(0, 3, 1, 2) * 2 - 1
    t_start, _ = img2img_timesteps(T, strength)
    m = mask_latents_ref(preprocess_mask_ref(mask, 64, 64), 4, 64, 64)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    res = []
    for ref, venc, dev, dt in oracles:
        procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

        def set_scale(s):
            for p in procs:
                p.scale = s
        with torch.no_grad():
            lat, img_lat, noise = prepare_inpaint_latents(lambda x: venc.encode(x.to(dt)), pix.to(dev), 4, _gens(),
                                                          t_start, T, strength, TINY_VAE.scaling_factor)
        fn = lambda s, t, e, te, ti: ref(s.to(dt), t, e, te, ti).to(torch.float16)  # noqa: E731
        res.append(inpaint_denoise_loop(fn, lat, img_lat, noise, m.to(dev), emb["prompt_embeds"].to(dev, dt),
                                        emb["negative_prompt_embeds"].to(dev, dt), emb["pooled_prompt_embeds"].to(dev, dt),
                                        emb["negative_pooled_prompt_embeds"].to(dev, dt), tid.to(dev), T, strength,
                                        guidance_scale=7.5, set_scale=set_scale, conditioning_scale=0.7,
                                        control_guidance_end=0.7).float().cpu())
    r, e = res
    e_nat, e_eag, mx = (o.float().cpu() - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    print(f"[inpaint tiny graph] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  max|ref| {mx:.3e}")
    assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)


def test_inpaint_bit_exact_invariants(pipes):
    """All-zero mask -> exactly the clean image latents.  All-one mask at strength 1 -> text-to-image from the same fp16
    noise (drawn after the posterior eps).  All-one mask at strength s < 1 with one generator -> image-to-image at s."""
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline, preprocess_image
    i2i, pipe, _ = pipes
    imgs, emb = _images(2, seed=3), _emb()
    common = dict(num_inference_steps=6, height=64, width=64, guidance_scale=7.5, control_guidance_end=0.7,
                  output_type="latent", **emb)
    pipe.set_scale(0.7)
    zero = pipe(image=imgs, mask_image=_mask(0), strength=0.5, generator=_gens(), **common).images
    pix = preprocess_image(imgs, 8, 64, 64)
    _, img_lat, _ = pipe.prepare_inpaint_latents(pix, 4, _gens(), 3, False)
    assert torch.equal(zero, img_lat)

    pipe.set_scale(0.7)
    one = pipe(image=imgs, mask_image=_mask(255), strength=1.0, generator=torch.Generator().manual_seed(9), **common).images
    g = torch.Generator().manual_seed(9)
    torch.randn((2, 4, 8, 8), generator=g, dtype=torch.float32)             # the posterior eps of the two images
    noise = torch.randn((4, 4, 8, 8), generator=g, dtype=torch.float16)
    t2i = StableDiffusionXLCustomPipeline(pipe.unet)
    t2i.set_scale(0.7)
    want = t2i(latents=noise, **common).images
    assert torch.equal(one, want)

    common.pop("height"), common.pop("width")
    pipe.set_scale(0.7)
    one = pipe(image=imgs, mask_image=_mask(255), strength=0.6, generator=torch.Generator().manual_seed(9), height=64,
               width=64, **common).images
    i2i.set_scale(0.7)
    want = i2i(image=imgs, strength=0.6, generator=torch.Generator().manual_seed(9), **common).images
    assert torch.equal(one, want)


def test_text_img2img_inpaint_alternate_on_one_engine(pipes):
    """Text-to-image, image-to-image and inpainting alternate on one engine: each bit-identical to a fresh engine's;
    image-to-image replays the text-to-image graphs, inpainting captures its own once, the text-to-image graph count does
    not change."""
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    _, pipe, _ = pipes
    imgs, mask, emb = _images(2), _mask(), _emb()
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    lat_t2i = (torch.randn(4, 4, 8, 8, generator=torch.Generator().manual_seed(5)) * 14.6).half()
    common = dict(num_inference_steps=6, guidance_scale=5.0, control_guidance_end=0.7, output_type="latent", **emb)

    def t2i():
        pipe.set_scale(0.7)
        return pipe.engine.run(lat_t2i, *emb.values(), tid, 6, guidance_scale=5.0, ip_scale=0.7, control_guidance_end=0.7)

    def img2img():
        pipe.set_scale(0.7)
        return StableDiffusionXLImg2ImgPipeline.__call__(pipe, image=imgs, strength=0.5, generator=_gens(),
                                                         **common).images

    def inpaint():
        pipe.set_scale(0.7)
        return pipe(image=imgs, mask_image=mask, strength=0.5, generator=_gens(), height=64, width=64, **common).images
    pipe._engine = None
    a1 = t2i()
    n_t2i = pipe.engine.graphs_captured
    b1 = img2img()
    assert pipe.engine.graphs_captured == n_t2i, "img2img must replay the text-to-image graphs"
    c1 = inpaint()
    n_all = pipe.engine.graphs_captured
    assert n_all > n_t2i
    a2, b2, c2 = t2i(), img2img(), inpaint()
    assert pipe.engine.graphs_captured == n_all, "no graph may be re-captured when the three alternate"
    fresh = []
    for fn in (t2i, img2img, inpaint):
        pipe._engine = None
        fresh.append(fn())
    torch.cuda.synchronize()
    assert torch.equal(a1, a2) and torch.equal(a1, fresh[0])
    assert torch.equal(b1, b2) and torch.equal(b1, fresh[1])
    assert torch.equal(c1, c2) and torch.equal(c1, fresh[2])
