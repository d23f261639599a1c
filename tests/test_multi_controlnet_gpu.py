"""GPU tests of Multi-ControlNet on the H100: the fused injection kernel (bit-exact against a torch fp16 restatement of
diffusers' sum), inert nets, graph replay against eager steps, graph keys per active subset, engine reuse across single
and multi calls, the trajectory and the SDXL UNet step against the restatement (tests/multi_controlnet_ref.py), and
IPAdapterXL with two control images."""
import pytest
import torch

from test_controlnet_gpu import SDXL_SKIPS, _bar, _ref_pair, _rand

pytestmark = pytest.mark.gpu


def _want(skips, res_per_net, scales_per_net, rows0):
    """diffusers: acc = fp16(r_0 * s_0); acc = fp16(acc + fp16(r_k * s_k)); skip = fp16(skip + acc)."""
    out = []
    for e, sk in enumerate(skips):
        acc = None
        for rs, sc in zip(res_per_net, scales_per_net):
            add = (rs[e].float() * float(sc[e])).half()
            acc = add if acc is None else acc + add
        w = sk.clone()
        w[rows0:] = w[rows0:] + acc.reshape(w[rows0:].shape)
        out.append(w)
    return out


@pytest.mark.parametrize("k", [2, 3, 8])
@pytest.mark.parametrize("guess", [False, True])
def test_multi_kernel_bit_exact_sdxl_shapes(k, guess):
    from imagharmony_b200 import ops
    g = torch.Generator().manual_seed(k)
    n = 1
    skips = [_rand(2 * n, s, s, c, g=g, scale=3.0) for s, c in SDXL_SKIPS]
    rows0 = n if guess else 0
    res = [[_rand((2 * n - rows0) * s * s, c, g=g, scale=2.0) for s, c in SDXL_SKIPS] for _ in range(k)]
    scales = [(torch.logspace(-1, 0, 10) * (0.3 + 0.2 * j) if guess else torch.full((10,), 0.65 - 0.1 * j)).float()
              for j in range(k)]
    want = _want(skips, res, scales, rows0)
    ptrs = [s.data_ptr() for s in skips]
    ops.controlnet_add_residuals_multi(skips, res, [s.cuda() for s in scales], [rows0 * s * s for s, _ in SDXL_SKIPS])
    torch.cuda.synchronize()
    assert [s.data_ptr() for s in skips] == ptrs
    for got, w in zip(skips, want):
        assert torch.equal(got, w)


def test_k1_bit_identical_to_single_injection_and_scale0_is_identity():
    from imagharmony_b200 import ops
    g = torch.Generator().manual_seed(11)
    skips = [_rand(2, s, s, c, g=g, scale=3.0) for s, c in SDXL_SKIPS]
    res = [_rand(2 * s * s, c, g=g, scale=2.0) for s, c in SDXL_SKIPS]
    scale = (torch.rand(10, generator=g) * 1.5).float().cuda()
    a, b = [s.clone() for s in skips], [s.clone() for s in skips]
    ops.controlnet_add_residuals(a, res, scale, [0] * 10)
    ops.controlnet_add_residuals_multi(b, [res], [scale], [0] * 10)
    c = [s.clone() for s in skips]
    zero = torch.zeros(10, dtype=torch.float32, device="cuda")
    ops.controlnet_add_residuals_multi(c, [res, res, res], [zero, zero, zero], [0] * 10)
    torch.cuda.synchronize()
    for x, y, z, s in zip(a, b, c, skips):
        assert torch.equal(x, y) and torch.equal(z, s)
    assert all(torch.equal(x, w) for x, w in zip(a, _want(skips, [res], [scale.cpu()], 0)))


def _pipe(nets_cfg=2, seed=0, cfg_u=None, cfg_c=None):
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    return StableDiffusionXLControlNetPipeline.from_random(cfg_u or TINY, [cfg_c or TINY_CONTROLNET] * nets_cfg,
                                                           seed=seed)


def _zero_convs(net):
    for z in list(net.controlnet_down_blocks) + [net.controlnet_mid_block]:
        z.weight.data.zero_()
        z.bias.data.zero_()
    net.finalize()


def _embeds(pipe, seed=9):
    gen = torch.Generator("cpu").manual_seed(seed)
    D, P = pipe.unet.config.cross_attention_dim, pipe.unet.config.pooled_embed_dim
    return dict(prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
                negative_prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
                pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(),
                negative_pooled_prompt_embeds=torch.randn(1, P, generator=gen).half())


def _call(pipe, image, T=4, seed=3, **kw):
    g = torch.Generator("cuda").manual_seed(seed)
    return pipe(image=image, num_inference_steps=T, generator=g, output_type="latent", **_embeds(pipe), **kw).images


def _imgs(k, seed=0):
    return [torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(seed + j)) for j in range(k)]


@pytest.mark.parametrize("place", [0, 1])
def test_inert_net_next_to_a_is_bit_identical_to_single_a(place):
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    base = _pipe(2)
    a, b = base.controlnet.nets
    _zero_convs(b)
    nets = [b, a] if place == 0 else [a, b]
    img_a, img_b = _imgs(2)
    multi = StableDiffusionXLControlNetPipeline(base.unet, nets)
    got = _call(multi, [img_b, img_a] if place == 0 else [img_a, img_b], controlnet_conditioning_scale=[0.8, 0.8])
    want = _call(StableDiffusionXLControlNetPipeline(base.unet, a), img_a, controlnet_conditioning_scale=0.8)
    assert torch.equal(got, want)


@pytest.mark.parametrize("sched", ["euler", "euler_a", "dpm"])
@pytest.mark.parametrize("opts", [dict(controlnet_conditioning_scale=[0.9, 0.6]),
                                  dict(guess_mode=True, controlnet_conditioning_scale=0.7),
                                  dict(control_guidance_start=[0.0, 0.25], control_guidance_end=[0.5, 1.0])])
def test_graph_replay_bit_identical_to_eager(sched, opts):
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    pipe = _pipe(seed=1)
    pipe.scheduler = {"euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
                      "dpm": DPMSolverMultistepScheduler}[sched]()
    imgs = _imgs(2, seed=2)
    graph = _call(pipe, imgs, T=8, **opts)
    if "control_guidance_start" in opts:            # subsets (0,), (0, 1), (1,)
        assert pipe.engine.graphs_captured == 3
        assert sorted(k[-1][2] for k in pipe.engine._graphs) == [(0,), (0, 1), (1,)]
    pipe.engine.use_cuda_graph = False
    eager = _call(pipe, imgs, T=8, **opts)
    assert torch.isfinite(graph).all() and torch.equal(graph, eager)


def _engine_args(unet, seed=4):
    g = torch.Generator("cpu").manual_seed(seed)
    D, P = unet.config.cross_attention_dim, unet.config.pooled_embed_dim
    lat = torch.randn(1, 4, 16, 16, generator=g).half()
    tid = torch.tensor([[128., 128, 0, 0, 128, 128]])
    return (lat, torch.randn(1, 77, D, generator=g).half(), torch.randn(1, 77, D, generator=g).half(),
            torch.randn(1, P, generator=g).half(), torch.randn(1, P, generator=g).half(), tid, 4)


def test_engine_alternating_single_and_multi_matches_fresh_engines():
    from imagharmony_b200.controlnet import ControlNetCall, controlnet_keep
    from imagharmony_b200.denoise import DenoiseEngine
    pipe = _pipe(seed=5)
    a, b = pipe.controlnet.nets
    img_a, img_b = (i.half() for i in _imgs(2, seed=6))
    single = ControlNetCall(a, img_a, 0.8, False, controlnet_keep(4, 0.0, 0.75))
    multi = [single, ControlNetCall(b, img_b, 0.5, False, controlnet_keep(4, 0.25, 1.0))]
    args = _engine_args(pipe.unet)
    eng = DenoiseEngine(pipe.unet)
    got = [eng.run(*args, controlnet=c) for c in (single, multi, single)]
    want = [DenoiseEngine(pipe.unet).run(*args, controlnet=c) for c in (single, multi)]
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]) and torch.equal(got[2], want[0])
    assert not torch.equal(want[0], want[1])


def test_scale_change_does_not_recapture_and_reload_recaptures_only_its_graphs():
    pipe = _pipe(seed=3)
    imgs = _imgs(2, seed=5)
    win = dict(control_guidance_start=[0.0, 0.25], control_guidance_end=[0.5, 1.0])
    x = _call(pipe, imgs, T=8, controlnet_conditioning_scale=[1.0, 1.0], **win)
    n = pipe.engine.graphs_captured
    y = _call(pipe, imgs, T=8, controlnet_conditioning_scale=[0.4, 0.9], **win)
    assert pipe.engine.graphs_captured == n and not torch.equal(x, y)
    pipe.engine.use_cuda_graph = False
    assert torch.equal(y, _call(pipe, imgs, T=8, controlnet_conditioning_scale=[0.4, 0.9], **win))
    pipe.engine.use_cuda_graph = True
    pipe.controlnet.nets[1].finalize()              # a weight reload of net 1: its two graphs, not net 0's alone
    _call(pipe, imgs, T=8, controlnet_conditioning_scale=[0.4, 0.9], **win)
    assert pipe.engine.graphs_captured == n + 2


@pytest.mark.parametrize("sched", ["euler", "euler_a"])
@pytest.mark.parametrize("opts", [dict(controlnet_conditioning_scale=[1.0, 0.6]), dict(guess_mode=True),
                                  dict(control_guidance_start=[0.0, 0.25], control_guidance_end=[0.75, 1.0])])
def test_tiny_two_net_trajectory_matches_oracle(opts, sched):
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from multi_controlnet_ref import multi_controlnet_denoise_loop
    from oracle.scheduler_ref import euler_tables
    pipe = _pipe(seed=2)
    if sched == "euler_a":
        pipe.scheduler = EulerAncestralDiscreteScheduler()
    usd = {k: v for k, v in pipe.unet.state_dict().items() if "processor" not in k}
    refs = {d: [_ref_pair(TINY, TINY_CONTROLNET, usd, net.state_dict(), d) for net in pipe.controlnet.nets]
            for d in (torch.float32, torch.float16)}
    imgs = _imgs(2, seed=4)
    T = 4
    got = _call(pipe, imgs, T=T, **opts).float()
    _, _, ins = euler_tables(T)
    e = _embeds(pipe)
    tid = torch.tensor([[128., 128, 0, 0, 128, 128]])
    outs = {}
    with torch.no_grad():
        for d, pairs in refs.items():
            g = torch.Generator("cuda").manual_seed(3)
            lat0 = (torch.randn((1, 4, 16, 16), generator=g, device="cuda") * ins).half()
            outs[d] = multi_controlnet_denoise_loop(
                pairs[0][0], [rc for _, rc in pairs], lat0.to(d), e["prompt_embeds"].cuda().to(d),
                e["negative_prompt_embeds"].cuda().to(d), e["pooled_prompt_embeds"].cuda().to(d),
                e["negative_pooled_prompt_embeds"].cuda().to(d), tid.cuda().to(d), [i.cuda().to(d) for i in imgs], T,
                conditioning_scale=opts.get("controlnet_conditioning_scale", 1.0),
                guess_mode=opts.get("guess_mode", False),
                control_guidance_start=opts.get("control_guidance_start", 0.0),
                control_guidance_end=opts.get("control_guidance_end", 1.0), scheduler=sched, generator=g).float()
    err, lim = _bar(got, outs[torch.float32], outs[torch.float16])
    assert err <= max(lim, 2e-2 * outs[torch.float32].abs().max().item()), (err, lim)


def test_sdxl_two_net_unet_step_matches_fp16_restatement():
    """One SDXL 1024^2 CFG UNet step with two nets' residuals (native ControlNets + fused injection) against the
    restatement in fp32 and fp16."""
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET
    from multi_controlnet_ref import multi_forward_ref
    pipe = _pipe(cfg_u=SDXL_BASE, cfg_c=SDXL_CONTROLNET, seed=5)
    nets = list(pipe.controlnet.nets)
    usd = {k: v for k, v in pipe.unet.state_dict().items() if "processor" not in k}
    g = torch.Generator().manual_seed(2)
    lat = 128
    sample = torch.randn(2, 4, lat, lat, generator=g).half().cuda()
    ehs = torch.randn(2, 77, SDXL_BASE.cross_attention_dim, generator=g).half().cuda()
    ehs_u = torch.cat([ehs, torch.zeros(2, 4, SDXL_BASE.cross_attention_dim).half().cuda()], 1)
    te = torch.randn(2, SDXL_BASE.pooled_embed_dim, generator=g).half().cuda()
    tid = torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * 2).cuda()
    imgs = [torch.rand(2, 3, 1024, 1024, generator=g).half().cuda() for _ in nets]
    scales = [0.8, 0.5]
    t = torch.full((2,), 501.0, device="cuda")
    with torch.no_grad():
        outs = [net(sample, t, ehs, controlnet_cond=im, conditioning_scale=s, text_embeds=te, time_ids=tid)
                for net, im, s in zip(nets, imgs, scales)]
        got = pipe.unet(sample, t, ehs_u, te, tid, controlnet_residuals=(outs, 0)).float()
        del outs
        ref = {}
        for dt in (torch.float32, torch.float16):
            pairs = [_ref_pair(SDXL_BASE, SDXL_CONTROLNET, usd, net.state_dict(), dt) for net in nets]
            down, mid = multi_forward_ref([rc for _, rc in pairs], sample.to(dt), 501.0, ehs.to(dt),
                                          [im.to(dt) for im in imgs], scales, te.to(dt), tid.to(dt))
            ref[dt] = pairs[0][0](sample.to(dt), 501.0, ehs_u.to(dt), te.to(dt), tid.to(dt),
                                  down_block_additional_residuals=down, mid_block_additional_residual=mid).float()
            del pairs, down, mid
            torch.cuda.empty_cache()
    err, lim = _bar(got, ref[torch.float32], ref[torch.float16])
    assert err <= lim, (err, lim)


def test_ip_adapter_generate_with_two_control_images_1024():
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET
    from ip_adapter.attention_processor import CNAttnProcessor2_0
    from ip_adapter.ip_adapter import IPAdapterXL
    pipe = _pipe(cfg_u=SDXL_BASE, cfg_c=SDXL_CONTROLNET)
    ip = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4)
    for net in pipe.controlnet.nets:
        assert all(isinstance(p, CNAttnProcessor2_0) and p.num_tokens == 4 for p in net.attn_processors.values())
    emb = torch.randn(1, SDXL_BASE.pooled_embed_dim, generator=torch.Generator().manual_seed(0))
    control = [torch.rand(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(j)) for j in (1, 2)]
    out = ip.generate(clip_image_embeds=emb, num_samples=1, seed=0, num_inference_steps=2, image=control,
                      controlnet_conditioning_scale=[0.5, 0.7], control_guidance_end=[1.0, 0.5],
                      output_type="latent")
    assert out.shape == (1, 4, 128, 128) and torch.isfinite(out).all()
