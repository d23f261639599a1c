"""CPU tests of Multi-ControlNet on the plain-PyTorch stand-in ops: MultiControlNetModel's residual sum and the
engine loop with 2 and 3 nets against the restatement of diffusers 0.30 (tests/multi_controlnet_ref.py), the alignment
of scales and guidance windows, per-net batch expansion, the IP-adapter processors on every net, and the refusals."""
import dataclasses

import pytest
import torch

import fake_ops_controlnet
import fake_ops_euler_a
import fake_ops_multi_controlnet
from test_controlnet_cpu import _after_latents, _cn_pair, _image
from test_wiring_cpu import _Empty32, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def mcp(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for mod in (fake_ops_controlnet, fake_ops_euler_a, fake_ops_multi_controlnet):
        for name in mod.NAMES:
            monkeypatch.setattr(real_ops, name, getattr(mod, name))
    yield


@pytest.mark.parametrize("guess", [False, True])
def test_multi_model_sum_matches_reference(mcp, guess):
    """MultiControlNetModel.forward (each net's scaled residuals, summed in net order) against diffusers'
    MultiControlNetModel.forward, two TINY nets with their own images and scales."""
    from imagharmony_b200.config import TINY_CONTROLNET
    from imagharmony_b200.controlnet import MultiControlNetModel
    from multi_controlnet_ref import multi_forward_ref
    (a, ra), (b, rb) = _cn_pair(TINY_CONTROLNET, 0), _cn_pair(TINY_CONTROLNET, 1)
    multi = MultiControlNetModel([a, b])
    assert isinstance(multi.nets, torch.nn.ModuleList) and list(multi.nets) == [a, b]
    sample, ehs, te, tid = _inputs(TINY_CONTROLNET, 1, 16)
    ehs = ehs[:, :77].contiguous()
    imgs, scales = [_image(2, 128, seed=4), _image(2, 128, seed=5)], [0.7, 0.4]
    with torch.no_grad():
        got = multi(sample, torch.full((2,), 321.0), ehs, imgs, scales, guess_mode=guess, text_embeds=te, time_ids=tid)
        down, mid = multi_forward_ref([ra, rb], sample, 321.0, ehs, imgs, scales, te, tid, guess_mode=guess)
    assert len(got) == 10
    for r, want in zip(got, down + [mid]):
        r = r.reshape(want.shape[0], want.shape[2], want.shape[3], -1).permute(0, 3, 1, 2)
        assert torch.allclose(r, want, rtol=1e-4, atol=1e-4), (r - want).abs().max()


def _pipe(k, seed=0):
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    pipe = StableDiffusionXLControlNetPipeline.from_random(TINY, [TINY_CONTROLNET] * k, seed=seed, device="cpu")
    for m in [pipe.unet] + list(pipe.controlnet.nets):
        m.float()
        m.finalize()
    return pipe


def _refs(pipe):
    from controlnet_ref import ControlNetRef, UNetResidualRef
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from oracle import adapter_ref as A
    ref_u = UNetResidualRef(TINY)
    A.install_processors(ref_u, TINY)
    ref_u.load_state_dict({k: v.float() for k, v in pipe.unet.state_dict().items()})
    torch.nn.ModuleList(p for p in ref_u.attn_processors.values() if hasattr(p, "to_k_ip")).load_state_dict(
        {k: v.float() for k, v in torch.nn.ModuleList(
            p for p in pipe.unet.attn_processors.values() if hasattr(p, "to_k_ip")).state_dict().items()})
    refs = []
    for net in pipe.controlnet.nets:
        rc = ControlNetRef(TINY_CONTROLNET)
        rc.load_state_dict({k: v.float() for k, v in net.state_dict().items()})
        rc.set_attn_processor({k: A.SelfAttnProcessorRef() for k in rc.attn_processors})
        refs.append(rc)
    return ref_u, refs


CASES = [
    (2, dict(controlnet_conditioning_scale=[0.8, 0.5], control_guidance_start=[0.0, 0.25],
             control_guidance_end=[0.5, 1.0])),
    (2, dict(guess_mode=True, controlnet_conditioning_scale=0.6, control_guidance_end=[0.75, 1.0])),
    (3, dict(controlnet_conditioning_scale=[1.0, 0.3, 0.6], control_guidance_start=[0.0, 0.25, 0.5],
             control_guidance_end=[0.75, 1.0, 1.0])),
    (2, dict(guidance_scale=1.0, control_guidance_start=0.25)),
]


@pytest.mark.parametrize("sched", ["euler", "euler_a"])
@pytest.mark.parametrize("k, opts", CASES)
def test_pipeline_loop_matches_reference(mcp, k, opts, sched):
    """The pipeline with 2 and 3 nets (eager engine steps, fp32 stand-in ops) against the restated diffusers loop in
    which the inactive nets run at scale 0: staggered windows, different scales, guess mode, no CFG.  The restatement
    gets the control images as the pipeline hands them to the ControlNets, in fp16."""
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from multi_controlnet_ref import multi_controlnet_denoise_loop
    from oracle.scheduler_ref import euler_tables
    pipe = _pipe(k)
    if sched == "euler_a":
        pipe.scheduler = EulerAncestralDiscreteScheduler()
    ref_u, ref_cs = _refs(pipe)
    n, lat, T = 1, 8, 4
    g = torch.Generator().manual_seed(7)
    pos, neg = torch.randn(n, 77, 128, generator=g), torch.randn(n, 77, 128, generator=g)
    pp, npool = torch.randn(n, 64, generator=g), torch.randn(n, 64, generator=g)
    imgs = [_image(1, 8 * lat, seed=4 + j) for j in range(k)]
    kw = dict(guidance_scale=5.0)
    kw.update(opts)
    with _Empty32():
        pipe.engine.use_cuda_graph = False
        out = pipe(prompt_embeds=pos, negative_prompt_embeds=neg, pooled_prompt_embeds=pp,
                   negative_pooled_prompt_embeds=npool, image=imgs, num_inference_steps=T,
                   generator=torch.Generator().manual_seed(11), output_type="latent", **kw).images
    _, _, ins = euler_tables(T)
    gen = torch.Generator().manual_seed(11)
    lat0 = torch.randn((n, 4, lat, lat), generator=gen) * ins
    tid = torch.tensor([[8. * lat, 8. * lat, 0., 0., 8. * lat, 8. * lat]])
    want = multi_controlnet_denoise_loop(
        ref_u, ref_cs, lat0, pos, neg, pp, npool, tid, [im.half().float() for im in imgs], T,
        guidance_scale=kw["guidance_scale"],
        conditioning_scale=kw.get("controlnet_conditioning_scale", 1.0), guess_mode=kw.get("guess_mode", False),
        control_guidance_start=kw.get("control_guidance_start", 0.0),
        control_guidance_end=kw.get("control_guidance_end", 1.0), scheduler=sched, generator=gen)
    # fp32 round-off of the stand-in ops grows to ~4e-3 at |latent| ~ 7 over the 4 steps with the larger residuals of
    # the second random net, and the Euler A step adds a gap of the same size with every net at scale 0
    atol = 5e-3
    assert torch.allclose(out.float(), want, rtol=1e-3, atol=atol), (out.float() - want).abs().max()


def test_list_of_one_call_equals_single_call(mcp):
    """A list with one ControlNetCall runs exactly the single-net loop."""
    from imagharmony_b200.controlnet import ControlNetCall, controlnet_keep
    pipe = _pipe(1)
    net = pipe.controlnet.nets[0]
    latents, ehs, te, tid = _inputs(pipe.unet.config, 1, 8)
    call = ControlNetCall(net, _image(1, 64), 0.7, False, controlnet_keep(4, 0.25, 1.0))
    pipe.engine.use_cuda_graph = False
    with _Empty32():
        runs = [pipe.engine.run(latents[:1], ehs[1:, :77], ehs[:1, :77], te[1:], te[:1], tid[:1], 4, controlnet=c)
                for c in (call, [call])]
    assert torch.equal(runs[0], runs[1])


def test_alignment_of_scales_and_windows(monkeypatch):
    """[3P] diffusers 0.30: a float scale is broadcast, scalar start / end become one entry per net (or the other
    list's length); each net gets its own keep list."""
    from imagharmony_b200.controlnet import ControlNetCall, controlnet_keep
    pipe = _pipe(3)
    seen = {}

    def run(lat, *a, controlnet=None, **k):
        seen["cn"] = controlnet
        return lat
    monkeypatch.setattr(pipe.engine, "run", run)
    imgs = [_image(1, 64, seed=j) for j in range(3)]
    for kw, scales, windows in (
            (dict(controlnet_conditioning_scale=0.4), [0.4] * 3, [(0.0, 1.0)] * 3),
            (dict(controlnet_conditioning_scale=[1.0, 0.5, 0.2], control_guidance_start=0.2), [1.0, 0.5, 0.2],
             [(0.2, 1.0)] * 3),
            (dict(control_guidance_start=[0.0, 0.2, 0.4], control_guidance_end=0.8), [1.0] * 3,
             [(0.0, 0.8), (0.2, 0.8), (0.4, 0.8)]),
            (dict(control_guidance_start=0.1, control_guidance_end=[0.5, 0.6, 0.7]), [1.0] * 3,
             [(0.1, 0.5), (0.1, 0.6), (0.1, 0.7)])):
        pipe(prompt="a", image=imgs, num_inference_steps=10, output_type="latent", guess_mode=True, **kw)
        cn = seen["cn"]
        assert isinstance(cn, list) and len(cn) == 3 and all(isinstance(c, ControlNetCall) for c in cn)
        assert [c.model for c in cn] == list(pipe.controlnet.nets)
        assert [c.conditioning_scale for c in cn] == scales and all(c.guess_mode for c in cn)
        assert [c.keep for c in cn] == [controlnet_keep(10, s, e) for s, e in windows]
        for c, im in zip(cn, imgs):
            assert torch.equal(c.image, im.half())


def test_per_net_batch_expansion(monkeypatch):
    """[3P] prepare_image per net: a single image is repeated to the whole batch, a batch of images (one per prompt)
    by num_images_per_prompt."""
    pipe = _pipe(2)
    seen = {}

    def run(lat, *a, controlnet=None, **k):
        seen["cn"], seen["n"] = controlnet, lat.shape[0]
        return lat
    monkeypatch.setattr(pipe.engine, "run", run)
    one = _image(1, 64, seed=1)
    two = torch.cat([_image(1, 64, seed=2), _image(1, 64, seed=3)])
    pipe(prompt=["a", "b"], image=[one, two], num_images_per_prompt=2, num_inference_steps=4, output_type="latent")
    a, b = seen["cn"]
    assert seen["n"] == 4
    assert torch.equal(a.image, one.repeat_interleave(4, dim=0).half())
    assert torch.equal(b.image, two.repeat_interleave(2, dim=0).half())


def test_refusals(mcp):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetCall, ControlNetModel, MultiControlNetModel
    from ip_adapter import MultiControlNetModel as Exported
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    assert Exported is MultiControlNetModel
    with torch.device("meta"):
        nets = [ControlNetModel(TINY_CONTROLNET) for _ in range(9)]
        wide = ControlNetModel(dataclasses.replace(TINY_CONTROLNET, block_out_channels=(64, 128, 128)))
    with pytest.raises(IHError, match="empty"):
        MultiControlNetModel([])
    with pytest.raises(IHError, match="at most 8"):
        MultiControlNetModel(nets)
    with pytest.raises(IHError, match="entry 1 is str, not a ControlNetModel"):
        MultiControlNetModel([nets[0], "canny"])
    with pytest.raises(IHError, match="block_out_channels"):
        MultiControlNetModel([nets[0], wide])
    with pytest.raises(IHError, match="Multi-ControlNet: entry 0 is NoneType"):
        StableDiffusionXLControlNetPipeline(None, [None, None])
    with pytest.raises(IHError, match="MultiControlNetModel"), torch.device("meta"):
        ControlNetModel([TINY_CONTROLNET, TINY_CONTROLNET])
    assert len(MultiControlNetModel(nets[:8]).nets) == 8

    pipe = _pipe(2)
    img = _image(1, 64)
    bad = [(TypeError, dict(image=img)),
           (ValueError, dict(image=[[img, img], [img, img]])),
           (ValueError, dict(image=[img])),
           (ValueError, dict(image=[img, img, img])),
           (ValueError, dict(image=[img, img], controlnet_conditioning_scale=[1.0])),
           (ValueError, dict(image=[img, img], controlnet_conditioning_scale=[[1.0], [1.0]])),
           (ValueError, dict(image=[img, img], control_guidance_start=[0.0, 0.1], control_guidance_end=[1.0])),
           (ValueError, dict(image=[img, img], control_guidance_start=[0.0, 0.1, 0.2])),
           (ValueError, dict(image=[img, img], control_guidance_start=[0.0, 0.6], control_guidance_end=[1.0, 0.5])),
           (ValueError, dict(image=[img, img], control_guidance_end=[1.0, 1.2])),
           (ValueError, dict(image=[img, img], control_guidance_start=[-0.1, 0.0])),
           (ValueError, dict(image=[img, _image(1, 72)]))]
    for exc, kw in bad:
        with pytest.raises(exc):
            pipe(prompt="a", num_inference_steps=4, output_type="latent", **kw)

    single = StableDiffusionXLControlNetPipeline(pipe.unet, pipe.controlnet.nets[0])
    with pytest.raises(IHError, match="Multi-ControlNet"):
        single(prompt="a", image=img, controlnet_conditioning_scale=[1.0], num_inference_steps=4)

    eng = pipe.engine
    eng.use_cuda_graph = False
    latents, ehs, te, tid = _inputs(pipe.unet.config, 1, 8)
    a, b = (ControlNetCall(m, img, 1.0, False) for m in pipe.controlnet.nets)
    args = (latents[:1], ehs[1:, :77], ehs[:1, :77], te[1:], te[:1], tid[:1], 4)
    with pytest.raises(IHError, match="guess_mode"):
        eng.run(*args, controlnet=[a, ControlNetCall(b.model, img, 1.0, True)])
    with pytest.raises(IHError, match="1 .. 8"):
        eng.run(*args, controlnet=[a] * 9)
    with pytest.raises(IHError, match="1 .. 8"):
        eng.run(*args, controlnet=[])
    for kw in (dict(begin_step=1), dict(start_step=1), dict(stop_after=2),
               dict(inpaint=(latents[:1], latents[:1], latents[:1, :1]))):
        with pytest.raises(IHError, match="controlnet"):
            eng.run(*args, controlnet=[a, b], **kw)


def test_ip_adapter_installs_cn_processors_on_every_net(mcp):
    from ip_adapter.attention_processor import CNAttnProcessor2_0
    from ip_adapter.ip_adapter import IPAdapterXL
    pipe = _pipe(2)
    epochs = [net.graph_epoch for net in pipe.controlnet.nets]
    IPAdapterXL(pipe, None, None, "cpu", num_tokens=4)
    seen = []
    for net, epoch in zip(pipe.controlnet.nets, epochs):
        procs = list(net.attn_processors.values())
        assert procs and all(isinstance(p, CNAttnProcessor2_0) and p.num_tokens == 4 for p in procs)
        assert net.graph_epoch > epoch
        seen.append(procs[0])
    assert seen[0] is not seen[1]                      # one processor per net, as the reference installs them
