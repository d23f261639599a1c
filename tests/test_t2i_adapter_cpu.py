"""CPU tests of the SDXL T2I-Adapter: the native T2IAdapter / MultiAdapter against the fp32 restatement of diffusers
(tests/t2i_adapter_ref.py) on the plain-PyTorch stand-in ops (tests/fake_ops*.py), the loader and its refusals, the
UNet's injection points, the engine's keep window and graph keys, the pipeline loop for every scheduler, the refusals
made before any work, and IPAdapterXL.generate through the adapter pipeline."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import fake_ops_dpm
import fake_ops_euler_a
import fake_ops_t2i_adapter
from test_wiring_cpu import _Empty32, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def tap(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for mod in (fake_ops_t2i_adapter, fake_ops_euler_a, fake_ops_dpm):
        for name in mod.NAMES:
            monkeypatch.setattr(real_ops, name, getattr(mod, name))
    yield


def _adapter_pair(cfg, seed, dtype=torch.float32):
    """(native T2IAdapter on the CPU in `dtype`, T2IAdapterRef in fp32) with the same random weights."""
    from imagharmony_b200.t2i_adapter import T2IAdapter
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from t2i_adapter_ref import T2IAdapterRef
    with torch.device("meta"):
        shapes = shapes_of(T2IAdapterRef(cfg))
    sd = random_state_dict(shapes, seed)
    native = T2IAdapter.from_state_dict(cfg, sd, device="cpu").to(dtype)
    native.finalize()
    ref = T2IAdapterRef(cfg)
    ref.load_state_dict({k: v.float() for k, v in sd.items()})
    return native, ref.eval()


def _img(n, c, h, w, seed=0):
    return torch.rand(n, c, h, w, generator=torch.Generator().manual_seed(seed))


def _nchw(f):
    return f.permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# model and loader
# ---------------------------------------------------------------------------------------------------------------------
def test_state_dict_keys_are_diffusers():
    from imagharmony_b200.config import SDXL_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import T2IAdapter
    from t2i_adapter_ref import T2IAdapterRef
    with torch.device("meta"):
        a, r = T2IAdapter(SDXL_T2I_ADAPTER), T2IAdapterRef(SDXL_T2I_ADAPTER)
    assert {k: tuple(v.shape) for k, v in a.state_dict().items()} == {k: tuple(v.shape) for k, v in r.state_dict().items()}
    keys = set(a.state_dict())
    assert "adapter.conv_in.weight" in keys and a.state_dict()["adapter.conv_in.weight"].shape == (320, 768, 3, 3)
    assert {"adapter.body.1.in_conv.weight", "adapter.body.2.in_conv.weight"} <= keys
    assert not any(k.startswith(("adapter.body.0.in_conv", "adapter.body.3.in_conv")) for k in keys)
    assert "adapter.body.3.resnets.1.block2.bias" in keys


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_from_pretrained_round_trip(tmp_path, fmt):
    from safetensors.torch import save_file
    from imagharmony_b200.config import TINY_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import T2IAdapter
    from imagharmony_b200.weights import random_state_dict, shapes_of
    cfg = dataclasses.replace(TINY_T2I_ADAPTER, in_channels=1)
    with torch.device("meta"):
        shapes = shapes_of(T2IAdapter(cfg))
    sd = {k: v.half() for k, v in random_state_dict(shapes, 5).items()}
    (tmp_path / "config.json").write_text(json.dumps({
        "_class_name": "T2IAdapter", "adapter_type": "full_adapter_xl", "channels": list(cfg.channels),
        "downscale_factor": 16, "in_channels": 1, "num_res_blocks": 2}))
    if fmt == "safetensors":
        save_file(sd, str(tmp_path / "diffusion_pytorch_model.safetensors"))
    else:
        torch.save(sd, str(tmp_path / "diffusion_pytorch_model.bin"))
    m = T2IAdapter.from_pretrained(str(tmp_path), device="cpu")
    assert m.config == cfg
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


@pytest.mark.parametrize("change,words", [
    (dict(adapter_type="full_adapter"), "SD1.5"), (dict(adapter_type="light_adapter"), "SD1.5"),
    (dict(adapter_type="other"), "unknown"), (dict(channels=(320, 640, 1280)), "channels"),
    (dict(channels=(320, 640, 640, 1280)), "channels"), (dict(channels=(96, 192, 384, 384)), "channels"),
    (dict(num_res_blocks=3), "num_res_blocks"), (dict(downscale_factor=8), "downscale_factor"),
    (dict(in_channels=4), "in_channels")])
def test_refused_configs(change, words):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import SDXL_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import T2IAdapter, config_from_diffusers
    with pytest.raises(IHError, match=words):
        with torch.device("meta"):
            T2IAdapter(dataclasses.replace(SDXL_T2I_ADAPTER, **change))
    meta = {"adapter_type": "full_adapter_xl", "channels": [320, 640, 1280, 1280], "downscale_factor": 16}
    meta.update({k: list(v) if isinstance(v, tuple) else v for k, v in change.items()})
    with pytest.raises(IHError, match=words):
        config_from_diffusers(meta)
    with pytest.raises(IHError, match="SD1.5"):        # diffusers' defaults: adapter_type "full_adapter"
        config_from_diffusers({"channels": [320, 640, 1280, 1280]})


def test_odd_grid_and_multi_adapter_mismatch_refused(tap):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import MultiAdapter
    a, _ = _adapter_pair(TINY_T2I_ADAPTER, 0)
    with pytest.raises(IHError, match="multiples of 32"):
        a(_img(1, 3, 48, 64))                           # a 3 x 4 grid: the average pool would need ceil_mode
    b, _ = _adapter_pair(dataclasses.replace(TINY_T2I_ADAPTER, channels=(128, 256, 512, 512)), 1)
    with pytest.raises(IHError, match="channels"):
        MultiAdapter([a, b])
    with pytest.raises(IHError, match="use a T2IAdapter"):
        MultiAdapter([a])
    with pytest.raises(IHError, match="at most 8"):
        MultiAdapter([a] * 9)


@pytest.mark.parametrize("widths,in_ch,size", [("tiny", 3, (64, 96)), ("tiny", 1, (96, 64)), ("sdxl", 3, (64, 64))])
def test_forward_matches_reference(tap, widths, in_ch, size):
    """TINY and SDXL widths at a small grid, fp32 stand-in ops, against PixelUnshuffle / AvgPool / 1x1 conv."""
    from imagharmony_b200.config import SDXL_T2I_ADAPTER, TINY_T2I_ADAPTER
    cfg = dataclasses.replace(TINY_T2I_ADAPTER if widths == "tiny" else SDXL_T2I_ADAPTER, in_channels=in_ch)
    native, ref = _adapter_pair(cfg, 3)
    x = _img(2, in_ch, *size, seed=1)
    with torch.no_grad():
        got, want = native(x), ref(x)
    assert [tuple(_nchw(g).shape) for g in got] == [tuple(w.shape) for w in want]
    h, w = size[0] // 16, size[1] // 16
    assert [tuple(g.shape[1:]) for g in got] == [(h, w, cfg.channels[0]), (h, w, cfg.channels[1]),
                                                 (h // 2, w // 2, cfg.channels[2]), (h // 2, w // 2, cfg.channels[3])]
    for g, wnt in zip(got, want):
        assert torch.allclose(_nchw(g), wnt, rtol=1e-4, atol=1e-4), (_nchw(g) - wnt).abs().max()


def test_pixel_unshuffle_channel_order():
    from imagharmony_b200.t2i_adapter import pixel_unshuffle_nhwc
    x = torch.arange(2 * 3 * 32 * 48, dtype=torch.float32).reshape(2, 3, 32, 48)
    assert torch.equal(_nchw(pixel_unshuffle_nhwc(x, 16)), torch.nn.PixelUnshuffle(16)(x))
    assert pixel_unshuffle_nhwc(x, 16)[1, 1, 2, 1 * 256 + 3 * 16 + 5] == x[1, 1, 16 + 3, 32 + 5]


def test_folded_pool_conv_equals_pool_then_conv_in_fp16():
    """The 2x2 window conv with w / 4 rounds once where AvgPool2d then the 1x1 conv round twice: within 2 fp16 ulps of
    the output, and equal to pool-then-conv in fp32 up to fp32 round-off."""
    import torch.nn.functional as F
    from fake_ops_img2img import conv3x3_down
    from imagharmony_b200.t2i_adapter import AdapterBlock
    from t2i_adapter_ref import fold_pool_conv_ref
    g = torch.Generator().manual_seed(4)
    blk = AdapterBlock(640, 1280, 0, down=True)
    blk.in_conv.weight.data = (torch.randn(1280, 640, 1, 1, generator=g) * 640 ** -0.5).half().float()
    blk.in_conv.bias.data = (torch.randn(1280, generator=g) * 0.1).half().float()
    blk.half().finalize()
    x = (torch.randn(2, 8, 6, 640, generator=g) * 2).half()
    got = conv3x3_down(x, blk._w_in, blk.in_conv.bias).float()                 # fp32 math, one fp16 rounding
    xn = x.float().permute(0, 3, 1, 2)
    w, b = blk.in_conv.weight.float(), blk.in_conv.bias.float()
    pooled16 = F.avg_pool2d(xn, 2, ceil_mode=True).half().float()             # diffusers' fp16 pool output
    want16 = F.conv2d(pooled16, w, b).half().float().permute(0, 2, 3, 1)
    exact = F.conv2d(F.avg_pool2d(xn.double(), 2), w.double(), b.double()).permute(0, 2, 3, 1)
    assert torch.allclose(fold_pool_conv_ref(xn, w, b).permute(0, 2, 3, 1).double(), exact, rtol=1e-5, atol=1e-5)
    ulp = torch.maximum(exact.abs(), torch.full_like(exact, 2 ** -14)) * 2 ** -10
    # w / 4 is exact in fp16 except where it is subnormal (|w| < 2^-12): then it is off by at most 2^-25
    sub = 2 ** -25 * F.conv2d(xn.abs().double(), torch.ones(1, 640, 2, 2, dtype=torch.float64), stride=2)
    sub = sub.permute(0, 2, 3, 1)
    assert ((got - exact).abs() <= 0.5 * ulp + sub + 1e-6 * ulp).all()       # one rounding of the (folded) value
    pool_err = 2 ** -11 * (pooled16.abs().double().permute(0, 2, 3, 1) @ w.double()[:, :, 0, 0].abs().t())
    assert ((got - want16).abs() <= ulp + sub + pool_err).all()              # diffusers' second rounding point
    assert (got != want16).any()                                              # ... which the fold does not have


# ---------------------------------------------------------------------------------------------------------------------
# UNet injection
# ---------------------------------------------------------------------------------------------------------------------
def _unet_pair(seed=0):
    from oracle import adapter_ref as A
    from t2i_adapter_ref import UNetAdapterRef
    from test_wiring_cpu import _build
    from imagharmony_b200.config import TINY
    native, _ = _build(TINY, seed)
    ref = UNetAdapterRef(TINY)
    A.install_processors(ref, TINY)
    ref.load_state_dict({k: v.float() for k, v in native.state_dict().items()})
    return native, ref.eval()


def _features(n, lat, seed=6, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    s = lat // 2
    return [torch.randn(n, s, s, 64, generator=g) * scale, torch.randn(n, s, s, 128, generator=g) * scale,
            torch.randn(n, s // 2, s // 2, 256, generator=g) * scale, torch.randn(n, s // 2, s // 2, 256, generator=g) * scale]


def test_adapter_targets_sdxl_and_refusals():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import SDXL_BASE, SDXL_REFINER
    from imagharmony_b200.unet import adapter_targets, require_adapter_shapes
    assert adapter_targets(SDXL_BASE, 128, 128) == [(64, 64, 320), (64, 64, 640), (32, 32, 1280), (32, 32, 1280)]
    sdxl = [(64, 64, 320), (64, 64, 640), (32, 32, 1280), (32, 32, 1280)]
    require_adapter_shapes(SDXL_BASE, 128, 128, sdxl)
    with pytest.raises(IHError, match="block_out_channels"):
        require_adapter_shapes(SDXL_REFINER, 128, 128, sdxl)                  # the refiner's widths start at 384
    with pytest.raises(IHError, match="injection points"):
        require_adapter_shapes(SDXL_BASE, 128, 128, sdxl[:3] + [(32, 32, 640)])
    with pytest.raises(IHError, match="injection points"):
        require_adapter_shapes(SDXL_BASE, 128, 96, sdxl)


@pytest.mark.parametrize("cfg_batch", [True, False])
def test_unet_injection_matches_reference(tap, cfg_batch):
    """diffusers' down_intrablock_additional_residuals (the in-place `sample +=` of the attention-free first block
    included) against the native UNet with the features of one CFG half added to each half."""
    native, ref = _unet_pair(1)
    n, lat = 1, 16
    sample, ehs, te, tid = _inputs(native.config, n, lat)
    if not cfg_batch:
        sample, ehs, te, tid = sample[:n], ehs[:n], te[:n], tid[:n]
    B = sample.shape[0]
    feats = _features(n, lat)
    s = 0.7
    state = [_nchw(f) * s for f in feats]
    state = [torch.cat([v] * (B // n)) for v in state]
    with torch.no_grad():
        want = ref(sample, 321.0, ehs, te, tid, down_intrablock_additional_residuals=[v.clone() for v in state])
        got = native(sample, torch.full((B,), 321.0), ehs, te, tid,
                     adapter_residuals=(feats, torch.full((2,), s)))
        plain = native(sample, torch.full((B,), 321.0), ehs, te, tid)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()
    assert (got - plain).abs().max() > 1e-2


def test_each_feature_changes_only_what_is_downstream(tap):
    """Feature k non-zero alone: the skips taken before its injection point are bit-identical to a run with zero
    features, the one at the point (the same tensor) and all later ones differ.  Skip indices (TINY): 3 = block 0's
    downsampler (feature 0), 5 = block 1's last attention (feature 1), 8 = block 2's last attention (feature 2); feature
    3 is added after the mid block, so no skip changes but the output does."""
    native, _ = _unet_pair(2)
    sample, ehs, te, tid = _inputs(native.config, 1, 16)
    seen = []
    up0 = native.up_blocks[0].forward

    def spy(x, temb, e, skips):
        seen.append(([s.clone() for s in skips], x.clone()))
        return up0(x, temb, e, skips)
    native.up_blocks[0].forward = spy
    zero = [torch.zeros_like(f) for f in _features(1, 16)]
    with torch.no_grad():
        base_out = native(sample, torch.full((2,), 321.0), ehs, te, tid, adapter_residuals=(zero, torch.ones(2)))
        plain_out = native(sample, torch.full((2,), 321.0), ehs, te, tid)
        assert torch.equal(base_out, plain_out)
        base_skips, base_mid = seen[0]
        for k, first in enumerate((3, 5, 8, 9)):
            feats = list(zero)
            feats[k] = _features(1, 16, seed=10 + k)[k]
            out = native(sample, torch.full((2,), 321.0), ehs, te, tid, adapter_residuals=(feats, torch.ones(2)))
            skips, mid = seen[-1]
            for i, (a, b) in enumerate(zip(skips, base_skips)):
                assert torch.equal(a, b) == (i < first), (k, i)
            assert not torch.equal(mid, base_mid) and not torch.equal(out, base_out)
    del native.up_blocks[0].forward


def test_no_adapter_launch_sequence_is_unchanged(tap, monkeypatch):
    """adapter_residuals=None makes exactly the op calls of a UNet call without the argument."""
    import imagharmony_b200.ops as real_ops
    native, _ = _unet_pair(3)
    sample, ehs, te, tid = _inputs(native.config, 1, 16)
    log = []
    for name in dir(real_ops):
        fn = getattr(real_ops, name)
        if callable(fn) and not name.startswith("_") and getattr(fn, "__module__", "").startswith(("fake_ops", "imag")):
            monkeypatch.setattr(real_ops, name, (lambda f, nm: lambda *a, **k: (log.append(nm), f(*a, **k))[1])(fn, name))
    with torch.no_grad():
        native(sample, torch.full((2,), 321.0), ehs, te, tid)           # prepares the step-invariant conditioning
        log.clear()
        native(sample, torch.full((2,), 321.0), ehs, te, tid)
        first = list(log)
        log.clear()
        native(sample, torch.full((2,), 321.0), ehs, te, tid, adapter_residuals=None)
    assert log == first and len(first) > 50
    log.clear()
    with torch.no_grad():
        native(sample, torch.full((2,), 321.0), ehs, te, tid, adapter_residuals=(_features(1, 16), torch.ones(2)))
    assert log.count("controlnet_add_residuals") == 4 and len(log) == len(first) + 4


# ---------------------------------------------------------------------------------------------------------------------
# engine and pipeline
# ---------------------------------------------------------------------------------------------------------------------
def _pipe(k=1, seed=0, dtype=torch.float32):
    from imagharmony_b200.config import TINY, TINY_T2I_ADAPTER
    from ip_adapter.custom_pipelines import StableDiffusionXLAdapterPipeline
    cfg = [TINY_T2I_ADAPTER] * k if k > 1 else TINY_T2I_ADAPTER
    pipe = StableDiffusionXLAdapterPipeline.from_random(TINY, cfg, seed=seed, device="cpu")
    adapters = list(pipe.adapter.adapters) if k > 1 else [pipe.adapter]
    for m in [pipe.unet] + adapters:
        m.to(dtype)
        m.finalize()
    return pipe


def _refs(pipe):
    from oracle import adapter_ref as A
    from imagharmony_b200.config import TINY, TINY_T2I_ADAPTER
    from t2i_adapter_ref import T2IAdapterRef, UNetAdapterRef
    ref_u = UNetAdapterRef(TINY)
    A.install_processors(ref_u, TINY)
    ref_u.load_state_dict({k: v.float() for k, v in pipe.unet.state_dict().items()})
    adapters = list(pipe.adapter.adapters) if hasattr(pipe.adapter, "adapters") else [pipe.adapter]
    refs = []
    for a in adapters:
        r = T2IAdapterRef(TINY_T2I_ADAPTER)
        r.load_state_dict({k: v.float() for k, v in a.state_dict().items()})
        refs.append(r.eval())
    return ref_u.eval(), refs


def _embeds(n=1, seed=7):
    g = torch.Generator().manual_seed(seed)
    return dict(prompt_embeds=torch.randn(n, 77, 128, generator=g), negative_prompt_embeds=torch.randn(n, 77, 128, generator=g),
                pooled_prompt_embeds=torch.randn(n, 64, generator=g), negative_pooled_prompt_embeds=torch.randn(n, 64, generator=g))


def _pil(n, size=64, mode="RGB", seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    shape = (size, size) if mode == "L" else (size, size, 3)
    return [Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8), mode) for _ in range(n)]


LOOP_CASES = [
    ("euler", 1, dict()),
    ("euler", 1, dict(adapter_conditioning_factor=0.5, adapter_conditioning_scale=0.6, denoising_end=0.6)),
    ("euler", 1, dict(guidance_scale=1.0, guidance_rescale=0.3)),
    ("euler", 1, dict(num_images_per_prompt=2, guidance_rescale=0.5)),
    ("euler_a", 1, dict(adapter_conditioning_factor=0.75, adapter_conditioning_scale=0.8)),
    ("dpm", 1, dict(adapter_conditioning_factor=0.5)),
    ("dpm", 1, dict(denoising_end=0.7, guidance_scale=1.0)),
    ("euler", 2, dict(adapter_conditioning_scale=[0.7, 0.4])),
    ("euler_a", 2, dict(adapter_conditioning_factor=0.5)),
]


@pytest.mark.parametrize("sched,k,opts", LOOP_CASES)
def test_pipeline_loop_matches_reference(tap, sched, k, opts):
    """The adapter pipeline (eager engine steps, fp32 stand-in ops) against the restated diffusers loop: the features
    scaled once, repeated per image and for CFG, cloned into the UNet at steps i < int(loop steps * factor)."""
    from dpm_ref import dpm_denoise_loop
    from euler_a_ref import euler_a_denoise_loop
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler
    from ip_adapter.custom_pipelines import preprocess_adapter_image
    from oracle.scheduler_ref import denoise_loop, denoising_end_steps, euler_tables
    from t2i_adapter_ref import adapter_state_ref, adapter_unet_fn, multi_adapter_ref
    pipe = _pipe(k)
    if sched == "euler_a":
        pipe.scheduler = EulerAncestralDiscreteScheduler()
    elif sched == "dpm":
        pipe.scheduler = DPMSolverMultistepScheduler()
    ref_u, ref_a = _refs(pipe)
    T, lat = 4, 8
    nipp = opts.get("num_images_per_prompt", 1)
    guidance = opts.get("guidance_scale", 5.0)
    images = [_pil(1, seed=j)[0] for j in range(k)]
    emb = _embeds(nipp)
    with _Empty32():
        pipe.engine.use_cuda_graph = False
        out = pipe(image=images if k > 1 else images[0], num_inference_steps=T,
                   generator=torch.Generator().manual_seed(11), output_type="latent", **emb, **opts).images
    xs = [preprocess_adapter_image(im, 64, 64) for im in images]
    with torch.no_grad():
        if k > 1:
            feats = multi_adapter_ref(ref_a, xs, opts.get("adapter_conditioning_scale", [1.0] * k))  # a float: broadcast
        else:
            feats = ref_a[0](xs[0])
    state = adapter_state_ref(feats, opts.get("adapter_conditioning_scale", 1.0), nipp, guidance > 1.0, multi=k > 1)
    gen = torch.Generator().manual_seed(11)
    ins = 1.0 if sched == "dpm" else (float(euler_tables(T)[2]) if sched == "euler" else pipe.scheduler.init_noise_sigma)
    lat0 = (torch.randn((nipp, 4, lat, lat), generator=gen) * ins).half().float()
    tid = torch.tensor([[8. * lat, 8. * lat, 0., 0., 8. * lat, 8. * lat]] * nipp)
    dend = opts.get("denoising_end")
    if sched == "dpm":
        from dpm_ref import denoising_end_steps as dpm_end_steps, dpm_tables
        loop_T = dpm_end_steps(dpm_tables(T)[0].tolist(), dend)
    else:
        loop_T = denoising_end_steps(T, dend)
    fn = adapter_unet_fn(ref_u, state, loop_T, opts.get("adapter_conditioning_factor", 1.0))
    common = dict(guidance_scale=guidance, guidance_rescale=opts.get("guidance_rescale", 0.0), denoising_end=dend)
    e = emb
    args = (lat0, e["prompt_embeds"], e["negative_prompt_embeds"], e["pooled_prompt_embeds"],
            e["negative_pooled_prompt_embeds"], tid, T)
    with torch.no_grad():
        if sched == "euler":
            want = denoise_loop(fn, *args, **common)
        elif sched == "euler_a":
            want = euler_a_denoise_loop(fn, *args, generator=gen, **common)
        else:
            want = dpm_denoise_loop(fn, *args, **common)
    assert out.shape == want.shape
    assert torch.allclose(out.float(), want, rtol=1e-3, atol=3e-3), (out.float() - want).abs().max()


def test_keep_window_and_denoising_end(tap, monkeypatch):
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from imagharmony_b200.t2i_adapter import adapter_keep
    assert adapter_keep(10, 10, 0.5) == [1.0] * 5 + [0.0] * 5
    assert adapter_keep(10, 7, 0.5) == [1.0] * 3 + [0.0] * 7                  # int(7 * 0.5) = 3
    assert adapter_keep(4, 4, 1.0) == [1.0] * 4 and adapter_keep(4, 4, 0.0) == [0.0] * 4
    pipe = _pipe()
    seen = {}

    def run(lat, *a, adapter=None, num_loop_steps=None, **k):
        seen.update(keep=list(adapter.keep), loop=num_loop_steps, scale=adapter.scale)
        return lat
    monkeypatch.setattr(pipe.engine, "run", run)
    pipe(image=_pil(1)[0], num_inference_steps=10, denoising_end=0.75, adapter_conditioning_factor=0.5,
         adapter_conditioning_scale=0.3, output_type="latent", **_embeds())
    s = EulerDiscreteScheduler()
    s.set_timesteps(10)
    loop = sum(1 for t in s.timesteps if t >= round(1000 - 0.75 * 1000))
    assert seen["loop"] == loop and seen["keep"] == adapter_keep(10, loop, 0.5) and seen["scale"] == 0.3


def test_graph_keys_reused_across_scales_and_images(tap, monkeypatch):
    """At most two step graphs per shape (features on / off); a new scale or adapter image captures none."""
    from imagharmony_b200.denoise import DenoiseEngine
    pipe = _pipe()
    captured = []

    class Eager:
        def __init__(self, eng, loop, cn, ad):
            self.args = (eng, loop, cn, ad)

        def replay(self):
            eng, loop, cn, ad = self.args
            eng._step(loop, cn, ad)

    def capture(self, loop, cn=None, adapter=False):
        captured.append(adapter)
        return Eager(self, loop, cn, adapter)
    monkeypatch.setattr(DenoiseEngine, "_capture", capture)
    eng = pipe.engine
    eng.use_cuda_graph = True
    outs = []
    with _Empty32():
        for scale, seed in ((1.0, 0), (0.4, 1), (0.9, 2)):
            outs.append(pipe(image=_pil(1, seed=seed)[0], num_inference_steps=4, adapter_conditioning_factor=0.5,
                             adapter_conditioning_scale=scale, generator=torch.Generator().manual_seed(3),
                             output_type="latent", **_embeds()).images)
    assert sorted(captured) == [False, True]
    assert not torch.equal(outs[0], outs[1])
    eng.use_cuda_graph = False
    with _Empty32():
        again = pipe(image=_pil(1, seed=2)[0], num_inference_steps=4, adapter_conditioning_factor=0.5,
                     adapter_conditioning_scale=0.9, generator=torch.Generator().manual_seed(3), output_type="latent",
                     **_embeds()).images
    assert torch.equal(again, outs[2])


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_engine_refusals_do_no_work(tap):
    """Every _EXCLUDES combination with the adapter, and the adapter's own checks, raise before any launch, static
    buffer or K/V buffer (as tests/test_run_refusals_cpu.py checks the other options)."""
    from test_run_refusals_cpu import _kv_buffers
    from imagharmony_b200 import ops
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.controlnet import ControlNetCall
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.t2i_adapter import AdapterCall
    pipe = _pipe()
    T, n, lat = 4, 1, 8
    latents, ehs, te, tid = _inputs(pipe.unet.config, n, lat)
    args = dict(latents=latents[:n], prompt_embeds=ehs[n:, :77], negative_prompt_embeds=ehs[:n, :77],
                pooled=te[n:], negative_pooled=te[:n], time_ids=tid[:n], num_inference_steps=T)
    feats = _features(n, lat)
    call = AdapterCall(feats, 0.5)
    x, mask = torch.zeros(n, 4, lat, lat), torch.zeros(n, 1, lat, lat)
    value = {"begin_step": 1, "inpaint": (x, x, mask), "unet_cond": (mask, x), "start_step": 1, "stop_after": 2,
             "controlnet": ControlNetCall(None, torch.zeros(n, 3, 64, 64))}
    calls = [({"adapter": call, o: v}, "adapter cannot be combined") for o, v in value.items()]
    calls += [({"adapter": AdapterCall(feats[:3] + [feats[2][..., :128].contiguous()])}, "injection points"),
              ({"adapter": AdapterCall(_features(n, 2 * lat))}, "injection points"),
              ({"adapter": AdapterCall([torch.cat([f, f]) for f in feats])}, "images for a batch"),
              ({"adapter": AdapterCall(feats, 1.0, [1.0] * (T - 1))}, "keep")]
    eng = DenoiseEngine(pipe.unet, use_cuda_graph=False)
    kv = _kv_buffers([pipe.unet])
    for kw, words in calls:
        launches = ops.launch_count()
        with pytest.raises(IHError, match=words):
            eng.run(**{**args, **kw})
        assert ops.launch_count() == launches, list(kw)
        assert not eng._pool and not eng._schedules, list(kw)
        assert _kv_buffers([pipe.unet]) == kv, list(kw)
    with _Empty32():
        eng.run(**args, adapter=call)
    assert eng._pool and _kv_buffers([pipe.unet]) > kv


@pytest.mark.parametrize("case", ["batch", "batch_nipp", "sigmas", "timesteps", "scale_list", "rgba", "tensor_size"])
def test_pipeline_refusals_before_any_work(tap, monkeypatch, case):
    from imagharmony_b200._lib import IHError
    pipe = _pipe()

    def no_work(*a, **k):
        raise AssertionError("work was done before the call was refused")
    monkeypatch.setattr(pipe, "encode_prompt", no_work)
    monkeypatch.setattr(pipe.adapter, "forward", no_work)
    kw = dict(image=_pil(1)[0], num_inference_steps=4, output_type="latent", **_embeds())
    if case == "batch":                  # one image, a prompt batch of 2 under CFG: diffusers cannot broadcast
        kw.update(_embeds(2))
    elif case == "batch_nipp":
        kw.update(image=_pil(2), num_images_per_prompt=2)
    elif case in ("sigmas", "timesteps"):
        kw[case] = [1.0, 0.5]
    elif case == "scale_list":
        kw["adapter_conditioning_scale"] = [0.5, 0.5]
    elif case == "rgba":
        from PIL import Image
        kw["image"] = Image.new("RGBA", (64, 64))
    else:
        kw["image"] = torch.rand(1, 3, 64, 64)
        kw.update(height=96, width=64)
    with pytest.raises(IHError):
        pipe(**kw)
    assert not pipe.engine._pool and not pipe.engine._schedules


def test_broadcast_cases_that_diffusers_allows(tap, monkeypatch):
    """One image per prompt (tiled per num_images_per_prompt as diffusers' repeat), and one image for a prompt batch
    without CFG; a grayscale image gives one channel."""
    from imagharmony_b200.config import TINY, TINY_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import T2IAdapter
    from ip_adapter.custom_pipelines import StableDiffusionXLAdapterPipeline, preprocess_adapter_image
    pipe = _pipe()
    seen = {}

    def run(lat, *a, adapter=None, **k):
        seen["features"] = adapter.features
        return lat
    monkeypatch.setattr(pipe.engine, "run", run)
    imgs = _pil(2, seed=3)
    pipe(image=imgs, num_images_per_prompt=2, num_inference_steps=4, output_type="latent", prompt=["a", "b"])
    f0 = pipe.adapter(preprocess_adapter_image(imgs, 64, 64))[0]
    assert torch.equal(seen["features"][0], torch.cat([f0, f0]))              # [a, b, a, b]
    pipe(image=imgs[0], guidance_scale=1.0, num_inference_steps=4, output_type="latent", **_embeds(3))
    assert seen["features"][0].shape[0] == 3
    gray = StableDiffusionXLAdapterPipeline(pipe.unet, T2IAdapter.from_random(
        dataclasses.replace(TINY_T2I_ADAPTER, in_channels=1), device="cpu").float())
    gray.adapter.finalize()
    monkeypatch.setattr(gray.engine, "run", run)
    gray(image=_pil(1, mode="L")[0], num_inference_steps=4, output_type="latent", **_embeds())
    assert preprocess_adapter_image(_pil(1, mode="L")[0], 64, 64).shape == (1, 1, 64, 64)
    assert TINY.block_out_channels == TINY_T2I_ADAPTER.channels[:3]


def test_default_height_width_rounds_to_the_downscale_factor():
    pipe = _pipe()
    assert pipe._default_height_width(None, None, _pil(1, size=100)) == (96, 96)
    assert pipe._default_height_width(None, 64, [torch.zeros(1, 3, 70, 130)]) == (64, 64)


def test_ip_adapter_generate_through_adapter_pipeline(tap):
    """IPAdapterXL(adapter pipe, ...).generate(pil_image / clip embeds, image=sketch, adapter_conditioning_scale=...)
    with no change to ip_adapter.py; one sketch per sample."""
    from ip_adapter import IPAdapterXL
    pipe = _pipe(dtype=torch.float16)
    ip_model = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4)
    emb = torch.randn(1, ip_model._clip_dim(), generator=torch.Generator().manual_seed(0))
    common = dict(clip_image_embeds=emb, prompt="a sketch", num_samples=2, num_inference_steps=3, seed=[7, 8],
                  output_type="latent", image=[_pil(1, seed=5)[0]] * 2)
    a = ip_model.generate(adapter_conditioning_scale=0.8, **common)
    b = ip_model.generate(adapter_conditioning_scale=0.0, **common)
    assert a.shape == (2, 4, 8, 8) and torch.isfinite(a.float()).all()
    assert (a.float() - b.float()).abs().max() > 1e-3


def test_graph_key_fields_and_positions(tap, monkeypatch):
    """The step-graph key names its fields, and the adapter flag leaves the older fields where positional readers find
    them: (n, h, w) in front, the inpainting flag second to last, the ControlNet part last.  tools/bench_inpaint.py's
    and tools/bench_t2i_adapter.py's graph selections (by field name) find their graphs."""
    from imagharmony_b200.denoise import DenoiseEngine, GraphKey
    pipe = _pipe()
    captured = []

    def capture(self, loop, cn=None, adapter=False):
        captured.append(adapter)
        return None
    monkeypatch.setattr(DenoiseEngine, "_capture", capture)
    monkeypatch.setattr(DenoiseEngine, "_restart", lambda *a, **k: None)
    eng = DenoiseEngine(pipe.unet, use_cuda_graph=False)
    eng.use_cuda_graph = True
    monkeypatch.setattr(eng, "_graphs", _NoReplay())
    T, n, lat = 4, 1, 8
    latents, ehs, te, tid = _inputs(pipe.unet.config, n, lat)
    args = (latents[:n], ehs[n:, :77], ehs[:n, :77], te[n:], te[:n], tid[:n], T)
    x, mask = torch.zeros(n, 4, lat, lat), torch.zeros(n, 1, lat, lat)
    from imagharmony_b200.t2i_adapter import AdapterCall
    with _Empty32():
        eng.run(*args)
        eng.run(*args, inpaint=(x, x, mask))
        eng.run(*args, adapter=AdapterCall(_features(n, lat), 0.5, [1.0, 1.0, 0.0, 0.0]))
    keys = list(eng._graphs)
    assert all(isinstance(k, GraphKey) for k in keys) and len(keys) == 3
    assert GraphKey._fields[:10] == ("n", "h", "w", "L", "T", "use_cfg", "guidance", "rescale", "scale", "kind")
    assert GraphKey._fields[-3:] == ("cond", "ib", "controlnet")
    for k in keys:
        assert k[:3] == (k.n, k.h, k.w) == (n, lat, lat) and k[-2] is k.ib and k[-1] is k.controlnet is None
    assert sorted((k.ib, k.adapter) for k in keys) == [(False, False), (False, True), (True, False)]
    assert {k.ib for k in keys} == {True, False}                                 # what bench_inpaint.py selects by
    assert {k.adapter for k in keys if (k.n, k.h, k.w, k.T) == (n, lat, lat, T)} == {False, True}


class _NoReplay(dict):
    """A graph table whose entries replay nothing (the test above checks keys only)."""

    def __setitem__(self, key, value):
        super().__setitem__(key, (_Nothing(), value[1]))


class _Nothing:
    def replay(self):
        pass
