"""GPU tests of image-to-image: the bottom/right-padded stride-2 conv and the posterior + add_noise kernel against torch,
the native VAE encoder against the fp32 oracle (tests/img2img_ref.py, [3P] restated, parity unpinned) with the bar of
test_vae_gpu.py, and the graph-replayed img2img pipeline against the oracle trajectory."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_kernels_gpu import check, ops, rnd  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,H,W,Cin,Cout,alpha,tile_n", [
    (1, 16, 16, 64, 64, 1.0, 0), (2, 34, 22, 128, 64, 1.0, 0), (1, 64, 64, 128, 128, 2.0 ** -7, 0),
    (2, 30, 50, 64, 192, 1.0, 128), (1, 128, 96, 256, 256, 1.0, 256), (2, 24, 40, 128, 128, 0.5, 64),
    (1, 256, 256, 128, 128, 1.0, 0),
])
def test_conv_down_kernel(ops, B, H, W, Cin, Cout, alpha, tile_n):  # noqa: F811
    x_nchw = rnd(B, Cin, H, W)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rnd(Cout)
    x = x_nchw.permute(0, 2, 3, 1).contiguous()
    out = ops.conv3x3_down(x, ops.pack_conv3x3_weight(w), b, alpha=alpha, tile_n=tile_n)
    ref = alpha * F.conv2d(F.pad(x_nchw.float(), (0, 1, 0, 1)), w.float(), None, stride=2) + b.float()[:, None, None]
    check(out, ref.permute(0, 2, 3, 1), f"conv3x3_down {B}x{H}x{W} {Cin}->{Cout} a{alpha} bn{tile_n}")


def _ulps(a, b):
    """|a - b| in units of the fp16 spacing at b, over the elements where b is finite."""
    keep = torch.isfinite(b)
    a, b = a.float()[keep], b.float()[keep]
    e = torch.floor(torch.log2(b.abs().clamp_min(2.0 ** -14)))
    return ((a - b).abs() / torch.exp2(e - 10)).max().item()


@pytest.mark.parametrize("eps_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("Bm,Be", [(2, 2), (2, 4), (1, 1)])
def test_posterior_noise_kernel(ops, eps_dtype, Bm, Be):  # noqa: F811
    """vs the torch restatement of the same rounding points (img2img_ref.posterior_noise_ref) on the GPU.  Expected
    bit-exact: every rounding point is an explicit fp16 / fp32 rounding in both, and fp16 x fp16 products are exact in
    fp32; the bar allows 1 fp16 ulp because the fp32 exp of torch and of the kernel may differ in the last bit.
    logvar reaches the upper clamp (std = e^10), where z leaves the fp16 range: those elements must be inf in both."""
    from img2img_ref import posterior_noise_ref
    B, C, h, w = 4, 4, 24, 40
    g = torch.Generator().manual_seed(Bm * 10 + Be)
    mom = torch.randn(Bm, h, w, 16, generator=g) * 2
    mom[..., 4:8] = torch.randn(Bm, h, w, 4, generator=g) * 15        # logvar through both clamp ends
    mom = mom.half().cuda()
    eps = torch.randn(Be, C, h, w, generator=g).to(eps_dtype).cuda()
    noise = torch.randn(B, C, h, w, generator=g).half().cuda()
    for sigma in (14.614647, 3.0742, 0.0292):
        out = ops.vae_posterior_noise(mom, eps, noise, C, 0.13025, sigma)
        ref = posterior_noise_ref(mom, eps, noise, C, 0.13025, sigma)
        assert out.dtype == ref.dtype == torch.float16 and out.shape == ref.shape == (B, C, h, w)
        exact = (out == ref).float().mean().item()
        u = _ulps(out, ref)
        print(f"[posterior+noise eps {eps_dtype} Bm{Bm} Be{Be} sigma {sigma}] bit-exact {exact:.6f}  max ulp {u}")
        assert torch.equal(torch.isfinite(out), torch.isfinite(ref)) and torch.isfinite(ref).float().mean() > 0.9
        assert u <= 1.0


def _encoders(cfg, seed, sd=None):
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    if sd is None:
        with torch.device("meta"):
            shapes = shapes_of(VAEEncoderRef(cfg))
        sd = random_state_dict(shapes, seed)
    native = AutoencoderKLEncoder.from_state_dict(cfg, sd, device="cuda")
    ref32 = VAEEncoderRef(cfg)
    ref32.load_state_dict({k: v.float() for k, v in sd.items()})
    eager16 = VAEEncoderRef(cfg)
    eager16.load_state_dict({k: v.float() for k, v in sd.items()})
    return native, ref32.eval(), eager16.half().cuda().eval()


def _check_encoder(cfg, seed, B, H, W, ref_device="cpu"):
    native, ref32, eager16 = _encoders(cfg, seed)
    x = (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1).half()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        r = ref32.to(ref_device).encode(x.float().to(ref_device)).cpu()
        ref32.cpu()
        e = eager16.encode(x.cuda()).float().cpu()
        o = native.encode(x.cuda()).float().cpu()
    torch.cuda.synchronize()
    e_nat, e_eag, mx = (o - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    print(f"[vae encoder {cfg.block_out_channels} B{B} {H}x{W}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  "
          f"max|ref| {mx:.3e}")
    assert o.shape == (B, 8, H // 8, W // 8) and torch.isfinite(o).all()
    assert e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)


def test_vae_encoder_tiny_matches_oracle():
    from imagharmony_b200.config import TINY_VAE
    _check_encoder(TINY_VAE, seed=5, B=2, H=64, W=64)
    _check_encoder(TINY_VAE, seed=6, B=1, H=96, W=80)          # 120 mid-block tokens: not a multiple of 128


def test_vae_encoder_sdxl_256_matches_oracle():
    from imagharmony_b200.config import SDXL_VAE
    _check_encoder(SDXL_VAE, seed=7, B=1, H=256, W=256)


def test_vae_encoder_sdxl_1024_matches_oracle():
    """1024^2: the blocked mid-block attention over 16384 tokens.  The fp32 oracle runs on the GPU here (TF32 off) to
    keep the test short; it is the same restatement as on the CPU."""
    from imagharmony_b200.config import SDXL_VAE
    _check_encoder(SDXL_VAE, seed=8, B=1, H=1024, W=1024, ref_device="cuda")


def test_vae_tiled_encode_matches_oracle():
    from img2img_ref import tiled_encode_ref
    from imagharmony_b200.config import TINY_VAE
    native, ref32, _ = _encoders(TINY_VAE, seed=9)
    native.use_tiling = True
    x = (torch.rand(1, 3, 104, 88, generator=torch.Generator().manual_seed(3)) * 2 - 1).half()
    with torch.no_grad():
        r = tiled_encode_ref(ref32, x.float())
        o = native.encode(x.cuda()).float().cpu()
    torch.cuda.synchronize()
    err, mx = (o - r).abs().max().item(), r.abs().max().item()
    print(f"[vae tiled encode] max|err| {err:.3e} max|ref| {mx:.3e}")
    assert o.shape == r.shape and torch.isfinite(o).all() and err <= 1e-2 * mx, (err, mx)


def test_vae_encoder_scaled_stream_survives_fp16_overflow():
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY_VAE as cfg
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(VAEEncoderRef(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, 11).items()}
    for k in ("encoder.conv_in.weight", "encoder.conv_in.bias"):
        sd[k] = (sd[k] * 3e5).half().float()
    ref32 = VAEEncoderRef(cfg)
    ref32.load_state_dict(sd)
    x = (torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(12)) * 2 - 1).half()
    with torch.no_grad():
        r = ref32.eval().encode(x.float())
        stream = ref32.encoder.conv_in(x.float())
    assert stream.abs().max() > 65504, "the test model must overflow fp16"
    native = AutoencoderKLEncoder.from_state_dict(cfg, sd, device="cuda")
    o = native.encode(x.cuda()).float().cpu()
    plain = AutoencoderKLEncoder.from_state_dict(cfg, sd, device="cuda", stream_scale=1.0).encode(x.cuda()).float().cpu()
    torch.cuda.synchronize()
    err, mx = (o - r).abs().max().item(), r.abs().max().item()
    print(f"[vae encoder scaled stream] stream max {stream.abs().max().item():.3e}: scaled max|err| {err:.3e} "
          f"(max|ref| {mx:.3e}); plain fp16 finite: {bool(torch.isfinite(plain).all())}")
    assert torch.isfinite(o).all() and err <= 1e-2 * mx, (err, mx)
    assert not torch.isfinite(plain).all(), "without the scaled stream this model overflows fp16"


def _pipe_and_oracles():
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    pipe = StableDiffusionXLImg2ImgPipeline.from_random(TINY, seed=0, device="cuda", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(procs), 1).items()})
    pipe.unet.finalize()
    sd = {k: v.float().cpu() for k, v in pipe.unet.state_dict().items()}
    vsd = {k: v.float().cpu() for k, v in pipe.vae_encoder.state_dict().items()}
    out = []
    for dev, dt in (("cpu", torch.float32), ("cuda", torch.float16)):
        ref = UNetRef(TINY)
        A.install_processors(ref, TINY)
        ref.load_state_dict(sd)
        venc = VAEEncoderRef(TINY_VAE)
        venc.load_state_dict(vsd)
        out.append((ref.to(dev, dt).eval(), venc.to(dev, dt).eval(), dev, dt))
    return pipe, out


def test_img2img_graph_replayed_matches_oracle_trajectory():
    """TINY UNet + TINY_VAE, CFG, IP scale 0.7 gated off for the last step, strength 0.5 of 6 steps, two images tiled
    to a prompt batch of four, graph-replayed -- vs the fp32 oracle trajectory, bar of SURVEY section 7 (native error at
    most twice the torch-fp16 eager path's, or 2e-3 of the reference's range).  Then text-to-image and img2img run
    alternately on one engine: both bit-identical to fresh engines, and img2img replays the text-to-image graphs."""
    from PIL import Image
    from img2img_ref import img2img_denoise_loop, img2img_timesteps, prepare_img2img_latents
    from imagharmony_b200.config import TINY, TINY_VAE
    from oracle.scheduler_ref import euler_tables
    pipe, oracles = _pipe_and_oracles()
    rng = np.random.default_rng(0)
    imgs = [Image.fromarray(rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)) for _ in range(2)]
    g = torch.Generator().manual_seed(11)
    pe, ne = (torch.randn(4, 81, TINY.cross_attention_dim, generator=g).half() for _ in range(2))
    pp, npool = (torch.randn(4, TINY.pooled_embed_dim, generator=g).half() for _ in range(2))
    T, strength = 6, 0.5
    emb = dict(prompt_embeds=pe, negative_prompt_embeds=ne, pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npool)

    def gens():
        return [torch.Generator().manual_seed(s) for s in (1, 2, 3, 4)]

    def img2img():
        pipe.set_scale(0.7)
        return pipe(image=imgs, strength=strength, num_inference_steps=T, guidance_scale=5.0, generator=gens(),
                    control_guidance_end=0.7, output_type="latent", **emb).images

    o = img2img()
    torch.cuda.synchronize()
    pix = torch.from_numpy(np.stack([np.array(im).astype(np.float32) / 255.0 for im in imgs])).permute(0, 3, 1, 2) * 2 - 1
    t_start, _ = img2img_timesteps(T, strength)
    sigma = float(euler_tables(T)[1][t_start])
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    res = []
    for ref, venc, dev, dt in oracles:
        procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

        def set_scale(s):
            for p in procs:
                p.scale = s
        with torch.no_grad():
            lat = prepare_img2img_latents(lambda x: venc.encode(x.to(dt)), pix.to(dev), 4, gens(), sigma,
                                          TINY_VAE.scaling_factor)
        fn = lambda s, t, e, te, ti: ref(s.to(dt), t, e, te, ti).to(torch.float16)  # noqa: E731
        res.append(img2img_denoise_loop(fn, lat, pe.to(dev, dt), ne.to(dev, dt), pp.to(dev, dt), npool.to(dev, dt),
                                        tid.to(dev), T, strength, guidance_scale=5.0, set_scale=set_scale,
                                        conditioning_scale=0.7, control_guidance_end=0.7).float().cpu())
    r, e = res
    e_nat, e_eag, mx = (o.float().cpu() - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    print(f"[img2img tiny graph] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  max|ref| {mx:.3e}")
    assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)

    # alternate text-to-image and img2img on one engine
    lat_t2i = (torch.randn(4, 4, 8, 8, generator=torch.Generator().manual_seed(5)) * 14.6).half()

    def t2i():
        pipe.set_scale(0.7)
        return pipe.engine.run(lat_t2i, pe, ne, pp, npool, tid, T, guidance_scale=5.0, ip_scale=0.7,
                               control_guidance_end=0.7)
    a1 = t2i()
    n_graphs = pipe.engine.graphs_captured
    b1 = img2img()
    assert pipe.engine.graphs_captured == n_graphs, "img2img must replay the text-to-image graphs"
    a2, b2 = t2i(), img2img()
    pipe._engine = None
    a_fresh = t2i()
    pipe._engine = None
    b_fresh = img2img()
    torch.cuda.synchronize()
    assert torch.equal(a1, a2) and torch.equal(a1, a_fresh)
    assert torch.equal(b1, b2) and torch.equal(b1, b_fresh) and torch.equal(b1, o)
