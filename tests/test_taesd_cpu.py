"""CPU tests of the native tiny autoencoder decoder (imagharmony_b200.taesd): diffusers' key schema and the folder
round trip, the config refusals, the decoder's wiring against the fp32 oracle (tests/taesd_ref.py) with stand-in ops,
the pipelines' output path and refusals, and the FLOP / byte counts of tools/bench_taesd.py."""
import dataclasses
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMALL = dict(num_decoder_blocks=(1, 2, 1, 1))       # four stages, fewer blocks: a quick CPU model


@pytest.fixture()
def taesd_ops(monkeypatch):
    import fake_ops
    import imagharmony_b200.ops as real_ops
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real_ops, name):
            monkeypatch.setattr(real_ops, name, getattr(fake_ops, name))
    yield


def _cfg(**kw):
    from imagharmony_b200.config import TAESDXL
    return dataclasses.replace(TAESDXL, **kw)


def _pair(cfg, seed=0):
    from imagharmony_b200.taesd import AutoencoderTinyDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from taesd_ref import AutoencoderTinyRef
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderTinyRef(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, seed).items()}
    ref = AutoencoderTinyRef(cfg)
    ref.load_state_dict(sd)
    with torch.device("meta"):
        native = AutoencoderTinyDecoder(cfg)
    native.load_state_dict(sd, assign=True)
    native.finalize()
    return native, ref.eval()


def test_key_schema_is_diffusers():
    from imagharmony_b200.config import TAESDXL
    from imagharmony_b200.taesd import AutoencoderTinyDecoder
    from imagharmony_b200.weights import shapes_of
    from taesd_ref import AutoencoderTinyRef
    with torch.device("meta"):
        native, ref = shapes_of(AutoencoderTinyDecoder(TAESDXL)), shapes_of(AutoencoderTinyRef(TAESDXL))
    assert native == ref
    want = {}
    for i in (0, 6, 11, 16, 18):
        want[f"decoder.layers.{i}.weight"] = (3 if i == 18 else 64, 4 if i == 0 else 64, 3, 3)
        if i in (0, 18):
            want[f"decoder.layers.{i}.bias"] = (3 if i == 18 else 64,)
    for k in (2, 3, 4, 7, 8, 9, 12, 13, 14, 17):
        for j in (0, 2, 4):
            want[f"decoder.layers.{k}.conv.{j}.weight"] = (64, 64, 3, 3)
            want[f"decoder.layers.{k}.conv.{j}.bias"] = (64,)
    assert native == want


def _write_folder(path, cfg, meta=None, seed=0, with_encoder=True):
    from safetensors.torch import save_file
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from taesd_ref import AutoencoderTinyRef
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderTinyRef(cfg))
    sd = random_state_dict(shapes, seed)
    if with_encoder:                                  # a full AutoencoderTiny checkpoint: the encoder is ignored
        sd["encoder.layers.0.weight"] = torch.zeros(64, 3, 3, 3, dtype=torch.float16)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(path, "diffusion_pytorch_model.safetensors"))
    m = {"_class_name": "AutoencoderTiny", "act_fn": "relu", "upsample_fn": "nearest", "upsampling_scaling_factor": 2,
         "latent_channels": cfg.latent_channels, "out_channels": cfg.out_channels,
         "decoder_block_out_channels": list(cfg.decoder_block_out_channels),
         "num_decoder_blocks": list(cfg.num_decoder_blocks), "scaling_factor": cfg.scaling_factor,
         "encoder_block_out_channels": [64, 64, 64, 64], "num_encoder_blocks": [1, 3, 3, 3]}
    m.update(meta or {})
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(m, f)
    return sd


def test_from_pretrained_round_trip(tmp_path):
    from imagharmony_b200.config import TAESDXL
    from ip_adapter import AutoencoderTiny
    sd = _write_folder(str(tmp_path), TAESDXL)
    m = AutoencoderTiny.from_pretrained(str(tmp_path), torch_dtype=torch.float16, device="cpu")
    assert m.config == TAESDXL
    own = m.state_dict()
    assert set(own) == {k for k in sd if k.startswith("decoder.")}
    for k, v in own.items():
        assert v.dtype == torch.float16 and torch.equal(v, sd[k]), k
    with pytest.raises(Exception):
        AutoencoderTiny.from_pretrained(str(tmp_path), torch_dtype=torch.float32, device="cpu")


@pytest.mark.parametrize("meta", [{"act_fn": "silu"}, {"upsample_fn": "bilinear"}, {"upsampling_scaling_factor": 4},
                                  {"decoder_block_out_channels": [96, 96, 96, 96]},
                                  {"decoder_block_out_channels": [64, 64, 128, 128]},
                                  {"num_decoder_blocks": [3, 3, 1]}])
def test_config_refusals(tmp_path, meta):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TAESDXL
    from ip_adapter import AutoencoderTiny
    _write_folder(str(tmp_path), TAESDXL, meta)
    with pytest.raises(IHError):
        AutoencoderTiny.from_pretrained(str(tmp_path), device="cpu")


@pytest.mark.parametrize("meta", [{"num_decoder_blocks": [3, 3, 3, 2]}, {"num_decoder_blocks": [1, 3, 3, 1]},
                                  {"decoder_block_out_channels": [128, 128, 128, 128]}])
def test_config_that_the_checkpoint_does_not_match_is_refused(tmp_path, meta):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TAESDXL
    from ip_adapter import AutoencoderTiny
    _write_folder(str(tmp_path), TAESDXL, meta)
    with pytest.raises(IHError, match="does not match"):
        AutoencoderTiny.from_pretrained(str(tmp_path), device="cpu")


@pytest.mark.parametrize("cfg_kw,shape", [({}, (2, 4, 5, 7)), (SMALL, (1, 4, 6, 4)),
                                          (dict(SMALL, scaling_factor=0.5), (1, 4, 3, 3))])
def test_decoder_wiring_matches_oracle(taesd_ops, cfg_kw, shape):
    import fake_ops
    cfg = _cfg(**cfg_kw)
    native, ref = _pair(cfg, seed=3)
    z = torch.randn(*shape, generator=torch.Generator().manual_seed(1)) * 4      # reaches into the tanh clamp
    fake_ops.launch_count_reset()
    with torch.no_grad():
        r = ref.decode(z)
        o = native.decode(z)
    B, _, h, w = shape
    assert o.shape == r.shape == (B, 3, 8 * h, 8 * w)
    assert torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()
    n = len(cfg.num_decoder_blocks)
    convs = 1 + 3 * sum(cfg.num_decoder_blocks) + (n - 1) + 1
    assert fake_ops.launch_count() == convs + (n - 1) + 2        # + upsamples + im2col and the NCHW gather


def _pipe_ns(vae):
    return SimpleNamespace(vae=vae, vae_decode=None)


@pytest.mark.parametrize("output_type", ["pil", "np", "pt"])
def test_pipeline_output_with_tiny_vae(taesd_ops, output_type):
    from imagharmony_b200.vae import postprocess
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    native, ref = _pair(_cfg(**SMALL), seed=4)
    z = torch.randn(2, 4, 4, 6, generator=torch.Generator().manual_seed(2))
    out = StableDiffusionXLCustomPipeline._output(_pipe_ns(native), z, output_type, True).images
    with torch.no_grad():
        want = postprocess(ref.decode(z), output_type)
    if output_type == "pil":
        assert len(out) == 2 and out[0].size == (48, 32)
        for a, b in zip(out, want):
            assert np.abs(np.asarray(a).astype(int) - np.asarray(b).astype(int)).max() <= 1
    else:
        assert tuple(out.shape) == tuple(want.shape)
        assert np.allclose(np.asarray(out), np.asarray(want), atol=1e-4)


def test_tiled_decode_is_refused(taesd_ops):
    from imagharmony_b200._lib import IHError
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    native, _ = _pair(_cfg(**SMALL), seed=5)
    pipe = _pipe_ns(native)
    StableDiffusionXLCustomPipeline.enable_vae_tiling(pipe)
    assert native.use_tiling
    with pytest.raises(IHError, match="tiled"):
        native.decode(torch.zeros(1, 4, 4, 4))


def _refusing(monkeypatch, pipe):
    """Every encoder and the prompt encoding raise if reached: a refusal must come before any work."""
    def boom(*a, **k):
        raise AssertionError("work was done before the refusal")
    if pipe.vae_encoder is not None:
        monkeypatch.setattr(pipe.vae_encoder, "encode_moments_nhwc", boom)
        monkeypatch.setattr(pipe.vae_encoder, "encode", boom)
    monkeypatch.setattr(pipe, "encode_prompt", boom)


def test_pixel_encode_with_tiny_vae_is_refused_before_any_work(taesd_ops, monkeypatch):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY, TINY_VAE
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline, StableDiffusionXLInpaintPipeline
    tiny, _ = _pair(_cfg(**SMALL), seed=6)
    init = torch.rand(1, 3, 64, 64) * 2 - 1
    for cls, kw in ((StableDiffusionXLImg2ImgPipeline, {}),
                    (StableDiffusionXLInpaintPipeline, dict(mask_image=torch.ones(1, 1, 64, 64), height=64, width=64))):
        pipe = cls.from_random(TINY, device="cpu", vae_cfg=TINY_VAE)
        pipe.vae = tiny
        _refusing(monkeypatch, pipe)
        with pytest.raises(IHError, match="tiny autoencoder"):
            pipe(prompt="a", image=init, strength=0.5, num_inference_steps=4, output_type="latent", **kw)


def test_latent_handoff_with_tiny_vae_needs_no_encoder(taesd_ops, monkeypatch):
    """`denoising_start` with latents encodes nothing: it runs with a tiny VAE and decodes through it."""
    from imagharmony_b200.config import TINY, TINY_VAE
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    tiny, ref = _pair(_cfg(**SMALL), seed=7)
    pipe = StableDiffusionXLImg2ImgPipeline.from_random(TINY, device="cpu", vae_cfg=TINY_VAE)
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict(random_state_dict(shapes_of(procs), 1))
    pipe.unet.finalize()
    pipe.vae = tiny

    def boom(*a, **k):
        raise AssertionError("the handoff must not encode")
    monkeypatch.setattr(pipe.vae_encoder, "encode_moments_nhwc", boom)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(3)).half()
    out = pipe(prompt="a", image=lat, denoising_start=0.5, num_inference_steps=4, output_type="latent").images
    img = pipe(prompt="a", image=lat, denoising_start=0.5, num_inference_steps=4, output_type="pt").images
    with torch.no_grad():
        want = (ref.decode(out.float()) / 2 + 0.5).clamp(0, 1)
    assert img.shape == (1, 3, 64, 64) and torch.allclose(img.float(), want, atol=1e-3)


def test_bench_tool_counts():
    """tools/bench_taesd.py: FLOPs against torch's FLOP counter on the oracles; bytes against a count by hand."""
    from torch.utils.flop_counter import FlopCounterMode
    from imagharmony_b200.config import SDXL_VAE, TAESDXL, TINY_VAE
    from oracle.vae_ref import VAEDecoderRef
    from taesd_ref import AutoencoderTinyRef
    from tools.bench_taesd import kl_cost, tiny_cost
    for cfg, model, cost, H, W in ((TAESDXL, AutoencoderTinyRef(TAESDXL), tiny_cost, 64, 48),
                                   (TINY_VAE, VAEDecoderRef(TINY_VAE), kl_cost, 64, 80)):
        with FlopCounterMode(display=False) as fc, torch.no_grad():
            model.decode(torch.randn(2, 4, H // 8, W // 8))
        assert cost(cfg, H, W, 2)[0] == fc.get_total_flops(), cfg
    f, b = tiny_cost(TAESDXL, 1024, 1024)
    assert 0.55e12 < f < 0.58e12                       # about 0.56 TFLOP per 1024^2 image
    assert 17 < kl_cost(SDXL_VAE, 1024, 1024)[0] / f < 20
    # bytes at a 1x1 latent: every launch's activations (fp16) and weights, counted by hand
    C = 64
    P = [1, 4, 16, 64]
    conv = lambda p, ci, co, bias=True: 2 * (p * ci + p * co + 9 * ci * co + (co if bias else 0))  # noqa: E731
    want = 2 * (4 + 2 * 64 + 64 * C + C + C)                                     # im2col + GEMM conv_in
    for i, nb in enumerate(TAESDXL.num_decoder_blocks):
        want += nb * (3 * conv(P[i], C, C) + 2 * P[i] * C)                       # blocks, residual read
        if i < 3:
            want += 2 * 5 * P[i] * C + conv(P[i + 1], C, C, bias=False)          # upsample + its conv
    want += conv(64, C, 3) + 2 * 64 * 13 + 2 * 64 * 19                          # conv_out (16 wide) + NCHW gather
    assert tiny_cost(TAESDXL, 8, 8)[1] == want
