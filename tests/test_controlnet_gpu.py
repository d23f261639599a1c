"""GPU tests of the SDXL ControlNet on the H100: the residual-injection kernel (bit-exact), the conditioning embedding,
the ControlNet forward and the UNet with residuals against the fp32 restatement of diffusers (tests/controlnet_ref.py),
the graph-replayed pipeline, re-capture rules, and IPAdapterXL on a ControlNet pipeline."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (side, C) of the 9 skips + the mid output at 1024^2: conv_in and level 0's two resnets, its downsampler, level 1's two
# transformers, its downsampler, level 2's two transformers, the mid block
SDXL_SKIPS = [(128, 320)] * 3 + [(64, 320)] + [(64, 640)] * 2 + [(32, 640)] + [(32, 1280)] * 3


def _rand(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


@pytest.mark.parametrize("guess", [False, True])
def test_injection_kernel_bit_exact_sdxl_shapes(guess):
    from imagharmony_b200 import ops
    g = torch.Generator().manual_seed(0)
    n = 1
    skips = [_rand(2 * n, s, s, c, g=g, scale=3.0) for s, c in SDXL_SKIPS]
    rows0 = n if guess else 0
    res = [_rand((2 * n - rows0) * s * s, c, g=g, scale=2.0) for s, c in SDXL_SKIPS]
    scale = (torch.logspace(-1, 0, 10) * 0.8 if guess else torch.full((10,), 0.65)).float()
    want = []
    for sk, r, (s, c), sc in zip(skips, res, SDXL_SKIPS, scale.tolist()):
        add = (r.float() * sc).half().reshape(2 * n - rows0, s, s, c)
        w = sk.clone()
        w[rows0:] = (w[rows0:].float() + add.float()).half()
        want.append(w)
    ptrs = [s.data_ptr() for s in skips]
    ops.controlnet_add_residuals(skips, res, scale.cuda(), [rows0 * s * s for s, _ in SDXL_SKIPS])
    torch.cuda.synchronize()
    assert [s.data_ptr() for s in skips] == ptrs
    for got, w in zip(skips, want):
        assert torch.equal(got, w)


@pytest.mark.parametrize("size", [(1024, 1024), (520, 776)])
def test_conditioning_embedding_matches_fp32(size):
    from imagharmony_b200.config import SDXL_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetConditioningEmbedding
    from imagharmony_b200.weights import random_state_dict, shapes_of
    emb = ControlNetConditioningEmbedding(320, 3, SDXL_CONTROLNET.conditioning_embedding_out_channels)
    sd = random_state_dict(shapes_of(emb), 3)
    emb.load_state_dict(sd)
    emb = emb.half().cuda()
    emb.finalize(bgr=False)
    img = torch.rand(2, 3, *size, generator=torch.Generator().manual_seed(1))
    got = emb(img.half().cuda()).float().cpu()
    x = F.silu(F.conv2d(img.half().float(), sd["conv_in.weight"].float(), sd["conv_in.bias"].float(), padding=1))
    for i in range(6):
        x = F.silu(F.conv2d(x, sd[f"blocks.{i}.weight"].float(), sd[f"blocks.{i}.bias"].float(), padding=1,
                            stride=1 + i % 2))
    want = F.conv2d(x, sd["conv_out.weight"].float(), sd["conv_out.bias"].float(), padding=1).permute(0, 2, 3, 1)
    assert got.shape == want.shape == (2, size[0] // 8, size[1] // 8, 320)
    err, mx = (got - want).abs().max().item(), want.abs().max().item()
    assert err <= 5e-3 * mx + 2e-3, (err, mx)


def _models(cfg_u, cfg_c, seed, device="cuda"):
    """native UNet + ControlNet (fp16, cuda) and their restatements in fp32 and fp16 (cuda)."""
    from controlnet_ref import ControlNetRef, UNetResidualRef
    from imagharmony_b200.controlnet import ControlNetModel
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        su, sc = shapes_of(UNetResidualRef(cfg_u)), shapes_of(ControlNetRef(cfg_c))
    usd, csd = random_state_dict(su, seed, device="cuda"), random_state_dict(sc, seed + 1, device="cuda")
    unet = UNet2DConditionModel.from_state_dict(cfg_u, usd)
    cn = ControlNetModel.from_state_dict(cfg_c, csd)
    return unet, cn, {dt: _ref_pair(cfg_u, cfg_c, usd, csd, dt) for dt in (torch.float32, torch.float16)}


def _ref_pair(cfg_u, cfg_c, usd, csd, dt):
    """(UNetResidualRef, ControlNetRef) on cuda in dtype dt; the UNet's IP weights zero like the native defaults."""
    from controlnet_ref import ControlNetRef, UNetResidualRef
    from oracle import adapter_ref as A
    ru, rc = UNetResidualRef(cfg_u), ControlNetRef(cfg_c)
    ru.load_state_dict({k: v.float() for k, v in usd.items()})
    for p in A.install_processors(ru, cfg_u).values():
        for q in p.parameters():
            q.data.zero_()
    rc.load_state_dict({k: v.float() for k, v in csd.items()})
    rc.set_attn_processor({k: A.SelfAttnProcessorRef() for k in rc.attn_processors})
    return ru.to("cuda", dt).eval(), rc.to("cuda", dt).eval()


def _bar(got, ref32, ref16):
    err = (got.float() - ref32).abs().max().item()
    e16 = (ref16.float() - ref32).abs().max().item()
    return err, max(2 * e16, 2e-3 * ref32.abs().max().item())


@pytest.mark.parametrize("size", ["tiny", "sdxl"])
def test_controlnet_and_unet_with_residuals_match_oracle(size):
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET, TINY, TINY_CONTROLNET
    cu, cc, lat = (TINY, TINY_CONTROLNET, 16) if size == "tiny" else (SDXL_BASE, SDXL_CONTROLNET, 128)
    unet, cn, refs = _models(cu, cc, 5)
    g = torch.Generator().manual_seed(2)
    sample = torch.randn(2, 4, lat, lat, generator=g).half().cuda()
    ehs = torch.randn(2, 77, cu.cross_attention_dim, generator=g).half().cuda()
    ehs_u = torch.cat([ehs, torch.randn(2, 4, cu.cross_attention_dim, generator=g).half().cuda()], 1)
    te = torch.randn(2, cu.pooled_embed_dim, generator=g).half().cuda()
    tid = torch.tensor([[8. * lat, 8. * lat, 0, 0, 8. * lat, 8. * lat]] * 2).cuda()
    img = torch.rand(2, 3, 8 * lat, 8 * lat, generator=g).half().cuda()
    with torch.no_grad():
        out = cn(sample, torch.full((2,), 501.0, device="cuda"), ehs, controlnet_cond=img, conditioning_scale=0.8,
                 text_embeds=te, time_ids=tid)
        got_res = [(r * s).half() for r, s in zip(out.residuals, out.scale)]
        ref = {}
        for dt, (ru, rc) in refs.items():
            down, mid = rc(sample.to(dt), 501.0, ehs.to(dt), img.to(dt), 0.8, te.to(dt), tid.to(dt))
            ref[dt] = (down + [mid], ru(sample.to(dt), 501.0, ehs_u.to(dt), te.to(dt), tid.to(dt),
                                        down_block_additional_residuals=down, mid_block_additional_residual=mid))
        for k, (gr, r32, r16) in enumerate(zip(got_res, ref[torch.float32][0], ref[torch.float16][0])):
            nchw = gr.reshape(r32.shape[0], r32.shape[2], r32.shape[3], -1).permute(0, 3, 1, 2)
            err, lim = _bar(nchw, r32, r16)
            assert err <= lim, (k, err, lim)
        noise = unet(sample, torch.full((2,), 501.0, device="cuda"), ehs_u, te, tid, controlnet_residuals=(out, 0))
        err, lim = _bar(noise, ref[torch.float32][1], ref[torch.float16][1])
        assert err <= lim, (err, lim)


def _pipe(seed=0, zero_zc=False, cfg_u=None, cfg_c=None):
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    pipe = StableDiffusionXLControlNetPipeline.from_random(cfg_u or TINY, cfg_c or TINY_CONTROLNET, seed=seed)
    if zero_zc:
        for z in list(pipe.controlnet.controlnet_down_blocks) + [pipe.controlnet.controlnet_mid_block]:
            z.weight.data.zero_()
            z.bias.data.zero_()
        pipe.controlnet.finalize()
    return pipe


def _call(pipe, img, T=4, seed=3, **kw):
    g = torch.Generator("cuda").manual_seed(seed)
    gen = torch.Generator("cpu").manual_seed(9)
    n, L, D = 1, 77, pipe.unet.config.cross_attention_dim
    emb = dict(prompt_embeds=torch.randn(n, L, D, generator=gen).half(),
               negative_prompt_embeds=torch.randn(n, L, D, generator=gen).half(),
               pooled_prompt_embeds=torch.randn(n, pipe.unet.config.pooled_embed_dim, generator=gen).half(),
               negative_pooled_prompt_embeds=torch.randn(n, pipe.unet.config.pooled_embed_dim, generator=gen).half())
    return pipe(image=img, num_inference_steps=T, generator=g, output_type="latent", **emb, **kw).images


@pytest.mark.parametrize("case", ["zero_convs", "scale0"])
def test_inert_controlnet_is_bit_identical_to_text_to_image(case):
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = _pipe(zero_zc=case == "zero_convs")
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(0))
    got = _call(pipe, img, controlnet_conditioning_scale=1.0 if case == "zero_convs" else 0.0)
    t2i = StableDiffusionXLCustomPipeline(pipe.unet)
    g = torch.Generator("cuda").manual_seed(3)
    gen = torch.Generator("cpu").manual_seed(9)
    D, P = pipe.unet.config.cross_attention_dim, pipe.unet.config.pooled_embed_dim
    want = t2i(prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
               negative_prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
               pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(),
               negative_pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(), height=128, width=128,
               num_inference_steps=4, generator=g, output_type="latent").images
    assert torch.equal(got, want)


@pytest.mark.parametrize("sched", ["euler", "euler_a", "dpm"])
@pytest.mark.parametrize("opts", [dict(), dict(guess_mode=True, controlnet_conditioning_scale=0.7),
                                  dict(control_guidance_start=0.25, control_guidance_end=0.75)])
def test_graph_replay_bit_identical_to_eager(sched, opts):
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    pipe = _pipe(seed=1)
    pipe.scheduler = {"euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
                      "dpm": DPMSolverMultistepScheduler}[sched]()
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    graph = _call(pipe, img, **opts)
    assert pipe.engine.graphs_captured >= 1
    pipe.engine.use_cuda_graph = False
    eager = _call(pipe, img, **opts)
    assert torch.isfinite(graph).all() and torch.equal(graph, eager)


@pytest.mark.parametrize("sched", ["euler", "euler_a"])
@pytest.mark.parametrize("opts", [dict(), dict(guess_mode=True), dict(control_guidance_start=0.25,
                                                                      control_guidance_end=0.75)])
def test_tiny_trajectory_matches_oracle(opts, sched):
    from controlnet_ref import controlnet_denoise_loop
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from oracle.scheduler_ref import euler_tables
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    pipe = _pipe(seed=2)
    if sched == "euler_a":
        pipe.scheduler = EulerAncestralDiscreteScheduler()
    usd = {k: v for k, v in pipe.unet.state_dict().items() if "processor" not in k}
    dt = {d: _ref_pair(TINY, TINY_CONTROLNET, usd, pipe.controlnet.state_dict(), d)
          for d in (torch.float32, torch.float16)}
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    T = 4
    got = _call(pipe, img, T=T, **opts).float()
    _, _, ins = euler_tables(T)
    gen = torch.Generator("cpu").manual_seed(9)
    D, P = TINY.cross_attention_dim, TINY.pooled_embed_dim
    pos, neg = torch.randn(1, 77, D, generator=gen).half(), torch.randn(1, 77, D, generator=gen).half()
    pp, npool = torch.randn(1, P, generator=gen).half(), torch.randn(1, P, generator=gen).half()
    tid = torch.tensor([[128., 128, 0, 0, 128, 128]])
    outs = {}
    with torch.no_grad():
        for d, (ru, rc) in dt.items():
            g = torch.Generator("cuda").manual_seed(3)                # _call's generator: latents, then step noise
            lat0 = (torch.randn((1, 4, 16, 16), generator=g, device="cuda") * ins).half()
            outs[d] = controlnet_denoise_loop(
                ru, rc, lat0.to(d), pos.cuda().to(d), neg.cuda().to(d), pp.cuda().to(d), npool.cuda().to(d),
                tid.cuda().to(d), img.cuda().to(d), T, guess_mode=opts.get("guess_mode", False),
                control_guidance_start=opts.get("control_guidance_start", 0.0),
                control_guidance_end=opts.get("control_guidance_end", 1.0), scheduler=sched, generator=g).float()
    err, lim = _bar(got, outs[torch.float32], outs[torch.float16])
    assert err <= max(lim, 2e-2 * outs[torch.float32].abs().max().item()), (err, lim)


def test_scale_change_does_not_recapture_and_reload_does():
    pipe = _pipe(seed=3)
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    a = _call(pipe, img, controlnet_conditioning_scale=1.0)
    n = pipe.engine.graphs_captured
    b = _call(pipe, img, controlnet_conditioning_scale=0.4)
    assert pipe.engine.graphs_captured == n and not torch.equal(a, b)
    pipe.engine.use_cuda_graph = False
    assert torch.equal(b, _call(pipe, img, controlnet_conditioning_scale=0.4))
    pipe.engine.use_cuda_graph = True
    pipe.controlnet.finalize()                      # a weight reload
    _call(pipe, img, controlnet_conditioning_scale=0.4)
    assert pipe.engine.graphs_captured > n


def test_ip_adapter_generate_with_control_image_1024():
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET
    from ip_adapter.ip_adapter import IPAdapterXL
    pipe = _pipe(cfg_u=SDXL_BASE, cfg_c=SDXL_CONTROLNET)
    ip = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4)
    emb = torch.randn(1, SDXL_BASE.pooled_embed_dim, generator=torch.Generator().manual_seed(0))
    control = torch.rand(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(1))
    out = ip.generate(clip_image_embeds=emb, num_samples=1, seed=0, num_inference_steps=2, image=control,
                      controlnet_conditioning_scale=0.5, output_type="latent")
    assert out.shape == (1, 4, 128, 128) and torch.isfinite(out).all()
