"""GPU tests of inpainting with the 9-channel inpainting UNet: the concatenating im2col kernel against the plain one on
the concatenated tensor, the 9-channel UNet forward against the fp32 oracle (TINY and SDXL-base at 1024^2), the
graph-replayed pipeline trajectory against the fp32 oracle with Euler and Euler Ancestral, bit-identity of graph
replay and eager steps, and the launch count of the step graph."""
import dataclasses

import numpy as np
import pytest
import torch

from test_kernels_gpu import ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kpad", [88, 128])
@pytest.mark.parametrize("B,H,W", [(1, 8, 8), (2, 17, 23), (3, 64, 48), (2, 128, 128), (1, 1, 5)])
def test_im2col_cat_kernel_equals_im2col_of_the_concatenation(ops, B, H, W, kpad):  # noqa: F811
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W)
    x0 = torch.randn(B, 4, H, W, generator=g).half().cuda()
    x1 = torch.randn(B, 5, H, W, generator=g).half().cuda()
    got = ops.im2col3x3_nchw_cat(x0, x1, kpad)
    want = ops.im2col3x3_nchw(torch.cat([x0, x1], 1).contiguous(), kpad)
    torch.cuda.synchronize()
    assert got.shape == want.shape == (B * H * W, kpad)
    assert torch.equal(got, want), (got.float() - want.float()).abs().max()
    assert not got[:, 81:].any()


def _pair9(cfg, seed, device_ref="cpu"):
    """(native 9-channel UNet, fp32 oracle on `device_ref`, fp16 eager oracle on the GPU) with identical weights."""
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    with torch.device("meta"):
        shapes = shapes_of(UNetRef(cfg))
    sd = random_state_dict(shapes, seed, device="cuda")
    native = UNet2DConditionModel.from_state_dict(cfg, sd, device="cuda")
    procs = torch.nn.ModuleList(native.attn_processors.values())
    ip_sd = random_state_dict(shapes_of(procs), seed + 1, device="cuda")
    procs.load_state_dict(ip_sd)
    native.finalize()

    def oracle(device, dtype):
        with torch.device("meta"):
            ref = UNetRef(cfg)
        ref = ref.to_empty(device=device)
        ref.load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in sd.items()})
        with torch.device("meta"):
            pr = A.install_processors(ref, cfg)
        for p in pr.values():
            p.to_empty(device=device)
        torch.nn.ModuleList(pr.values()).load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in ip_sd.items()})
        return ref.to(dtype).eval()
    return native, oracle(device_ref, torch.float32), oracle("cuda", torch.float16)


@pytest.mark.parametrize("which", ["tiny", "sdxl_1024"])
def test_unet9_forward_matches_oracle(which):
    """One forward of the 9-channel UNet (latents + cond through im2col3x3_nchw_cat and the K = 128 GEMM) vs the fp32
    oracle on the concatenated input, with the bar of test_unet_gpu.py (SURVEY section 7).  At SDXL-base 1024^2 (UNet
    batch 2) the fp32 oracle runs on the GPU with TF32 off to keep the test short."""
    from imagharmony_b200.config import SDXL_BASE, TINY
    cfg, lat, t, dev = ((TINY, 32, 601.0, "cpu") if which == "tiny" else (SDXL_BASE, 128, 481.0, "cuda"))
    cfg = dataclasses.replace(cfg, in_channels=9)
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    native, ref32, eager16 = _pair9(cfg, 21, dev)
    g = torch.Generator().manual_seed(5)
    B = 2
    x = torch.randn(B, 4, lat, lat, generator=g).half()
    cond = torch.cat([(torch.rand(B, 1, lat, lat, generator=g) > 0.5).float(),
                      torch.randn(B, 4, lat, lat, generator=g)], 1).half()
    ehs = torch.randn(B, 77 + cfg.num_ip_tokens, cfg.cross_attention_dim, generator=g).half()
    te = torch.randn(B, cfg.pooled_embed_dim, generator=g).half()
    tid = torch.tensor([[lat * 8.0, lat * 8.0, 0.0, 0.0, lat * 8.0, lat * 8.0]] * B)
    full = torch.cat([x, cond], 1)
    with torch.no_grad():
        r = ref32(full.float().to(dev), t, ehs.float().to(dev), te.float().to(dev), tid.to(dev)).float().cpu()
        e = eager16(full.cuda(), t, ehs.cuda(), te.cuda(), tid.cuda()).float().cpu()
        o = native(x.cuda(), torch.full((B,), t, device="cuda"), ehs.cuda(), te.cuda(), tid.cuda(),
                   cond=cond.cuda()).float().cpu()
    torch.cuda.synchronize()
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    e_nat, e_eag, mx = (o - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    print(f"[unet9 {which} B{B} {lat}^2] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  max|ref| {mx:.3e}")
    assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
    del native, ref32, eager16
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def pipe9():
    """TINY 9-channel UNet + TINY_VAE pipeline, and the (fp32 CPU, fp16 GPU) oracle pairs of UNet and VAE encoder."""
    from img2img_ref import VAEEncoderRef
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef
    cfg = dataclasses.replace(TINY, in_channels=9)
    pipe = StableDiffusionXLInpaintPipeline.from_random(cfg, seed=0, device="cuda", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(procs), 1).items()})
    pipe.unet.finalize()
    sd = {k: v.float().cpu() for k, v in pipe.unet.state_dict().items()}
    vsd = {k: v.float().cpu() for k, v in pipe.vae_encoder.state_dict().items()}
    oracles = []
    for dev, dt in (("cpu", torch.float32), ("cuda", torch.float16)):
        ref = UNetRef(cfg)
        A.install_processors(ref, cfg)
        ref.load_state_dict(sd)
        venc = VAEEncoderRef(TINY_VAE)
        venc.load_state_dict(vsd)
        oracles.append((ref.to(dev, dt).eval(), venc.to(dev, dt).eval(), dev, dt))
    return pipe, oracles


def _images(n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    return [Image.fromarray(rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)) for _ in range(n)]


def _mask():
    from PIL import Image
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


@pytest.mark.parametrize("strength", [0.5, 1.0])
@pytest.mark.parametrize("euler_a", [False, True])
def test_inpaint9_graph_replayed_matches_oracle_trajectory(pipe9, euler_a, strength):
    """TINY 9-channel UNet + TINY_VAE, CFG 7.5, IP scale 0.7 gated off for the last step, 6 steps, two images and one
    mask tiled to a prompt batch of four, a list of generators, graph-replayed -- vs the fp32 oracle trajectory with the
    bar of SURVEY section 7; and bit-identical to the same engine stepping eagerly (use_cuda_graph=False)."""
    from euler_a_ref import euler_a_denoise_loop
    from img2img_ref import img2img_denoise_loop, img2img_timesteps
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler, EulerDiscreteScheduler
    from inpaint_ref import preprocess_mask_ref
    from inpaint9_ref import prepare_inpaint9_inputs, unet9_fn
    pipe, oracles = pipe9
    pipe.scheduler = EulerAncestralDiscreteScheduler() if euler_a else EulerDiscreteScheduler()
    imgs, mask, emb = _images(2), _mask(), _emb()
    T = 6

    def run():
        pipe.set_scale(0.7)
        return pipe(image=imgs, mask_image=mask, strength=strength, num_inference_steps=T, height=64, width=64,
                    generator=_gens(), control_guidance_end=0.7, output_type="latent", **emb).images
    o = run()
    assert pipe.engine.use_cuda_graph and pipe.engine.graphs_captured > 0
    pipe._engine = DenoiseEngine(pipe.unet, use_cuda_graph=False, scheduler=pipe.scheduler)
    o_eager = run()
    pipe._engine = None
    torch.cuda.synchronize()
    assert torch.equal(o, o_eager), (o.float() - o_eager.float()).abs().max()
    pix = torch.from_numpy(np.stack([np.array(im).astype(np.float32) / 255.0 for im in imgs])).permute(0, 3, 1, 2) * 2 - 1
    t_start, _ = img2img_timesteps(T, strength)
    m = preprocess_mask_ref(mask, 64, 64)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 4)
    res = []
    for ref, venc, dev, dt in oracles:
        procs = [p for p in ref.attn_processors.values() if hasattr(p, "to_k_ip")]

        def set_scale(s):
            for p in procs:
                p.scale = s
        g = _gens()
        with torch.no_grad():
            lat, ml, mil = prepare_inpaint9_inputs(lambda x: venc.encode(x.to(dt)), pix.to(dev), m.to(dev), 4, g,
                                                   t_start, T, strength, TINY_VAE.scaling_factor)
        fn = unet9_fn(lambda s, t, e, te, ti: ref(s.to(dt), t, e, te, ti).to(torch.float16), ml, mil, True)
        embd = [emb[k].to(dev, dt) for k in ("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                                            "negative_pooled_prompt_embeds")]
        common = dict(guidance_scale=7.5, set_scale=set_scale, conditioning_scale=0.7, control_guidance_end=0.7)
        if euler_a:
            r = euler_a_denoise_loop(fn, lat.to(dev), *embd, tid.to(dev), T, generator=g, begin=t_start, **common)
        else:
            r = img2img_denoise_loop(fn, lat.to(dev), *embd, tid.to(dev), T, strength, **common)
        res.append(r.float().cpu())
    r, e = res
    e_nat, e_eag, mx = (o.float().cpu() - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    print(f"[inpaint9 tiny graph euler_a={euler_a} strength={strength}] native err {e_nat:.3e}  eager-fp16 err "
          f"{e_eag:.3e}  max|ref| {mx:.3e}")
    assert torch.isfinite(o).all() and e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)


def test_inpaint9_step_graph_has_the_text_to_image_launch_count(pipe9):
    """The 9-channel step reads its extra input in conv_in's im2col: same launch count as the 4-channel text-to-image
    step graph of the same architecture, shape, CFG and scheduler."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    pipe, _ = pipe9
    pipe.scheduler = EulerDiscreteScheduler()
    with torch.device("meta"):
        shapes = shapes_of(UNet2DConditionModel(TINY))
    unet4 = UNet2DConditionModel.from_state_dict(TINY, random_state_dict(shapes, 3, device="cuda"), device="cuda")
    emb = _emb(2)
    args = (emb["prompt_embeds"], emb["negative_prompt_embeds"], emb["pooled_prompt_embeds"],
            emb["negative_pooled_prompt_embeds"], torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2), 4)
    lat = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(0)).half()
    e4 = DenoiseEngine(unet4)
    e4.run(lat, *args, guidance_scale=5.0)
    e9 = DenoiseEngine(pipe.unet, scheduler=pipe.scheduler)
    e9.run(lat, *args, guidance_scale=5.0, begin_step=1,
           unet_cond=(torch.ones(2, 1, 8, 8, dtype=torch.float16), torch.zeros(2, 4, 8, 8, dtype=torch.float16)))
    torch.cuda.synchronize()
    print(f"[inpaint9 launches] 4-channel text-to-image {e4.last_launches_per_step}, 9-channel inpaint "
          f"{e9.last_launches_per_step} per step")
    assert e9.graphs_captured == e4.graphs_captured == 1
    assert e9.last_launches_per_step == e4.last_launches_per_step > 0
