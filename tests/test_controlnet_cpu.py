"""CPU tests of the SDXL ControlNet: the native ControlNetModel and the UNet's residual injection against the
restatement of diffusers (tests/controlnet_ref.py) on the plain-PyTorch stand-in ops (tests/fake_ops*.py), the
state-dict names, from_pretrained, the control-image preprocessing, the keep window and scales, the engine loop, the
IP-adapter processors on the ControlNet, and the refusals."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import fake_ops_controlnet
import fake_ops_euler_a
from test_wiring_cpu import _build, _Empty32, _inputs, patched  # noqa: F401  (fixture)


@pytest.fixture()
def cnp(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for mod in (fake_ops_controlnet, fake_ops_euler_a):
        for name in mod.NAMES:
            monkeypatch.setattr(real_ops, name, getattr(mod, name))
    yield


def _cn_pair(cfg, seed, zero_zc=False):
    """(native ControlNetModel in fp32 on the CPU, ControlNetRef) with the same random weights."""
    from controlnet_ref import ControlNetRef
    from imagharmony_b200.controlnet import ControlNetModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(ControlNetRef(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, seed).items()}
    if zero_zc:
        sd = {k: (torch.zeros_like(v) if k.startswith(("controlnet_down_blocks", "controlnet_mid_block")) else v)
              for k, v in sd.items()}
    with torch.device("meta"):
        native = ControlNetModel(cfg)
    native.load_state_dict(sd, assign=True)
    native.install_default_processors()
    native.finalize()
    ref = ControlNetRef(cfg)
    ref.load_state_dict(sd)
    from oracle import adapter_ref as A
    ref.set_attn_processor({k: A.SelfAttnProcessorRef() for k in ref.attn_processors})
    return native, ref.eval()


def _image(n, size, seed=4):
    return torch.rand(n, 3, size, size, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("order", ["rgb", "bgr"])
def test_controlnet_residuals_match_reference(cnp, order):
    """All 10 residuals of the TINY ControlNet (CFG batch of 2), unscaled, and the scale vector in and out of guess
    mode, against diffusers' scaled residuals."""
    from imagharmony_b200.config import TINY_CONTROLNET
    cfg = dataclasses.replace(TINY_CONTROLNET, controlnet_conditioning_channel_order=order)
    native, ref = _cn_pair(cfg, 0)
    sample, ehs, te, tid = _inputs(cfg, 1, 16)
    ehs = ehs[:, :77].contiguous()                    # a ControlNet without an IP adapter sees text tokens only
    img = _image(2, 128)
    with torch.no_grad():
        for guess, cs in ((False, 0.7), (True, 0.5)):
            out = native(sample, torch.full((2,), 321.0), ehs, controlnet_cond=img, conditioning_scale=cs,
                         guess_mode=guess, text_embeds=te, time_ids=tid)
            down, mid = ref(sample, 321.0, ehs, img, cs, te, tid, guess_mode=guess)
            assert len(out.residuals) == 10 and out.scale.dtype == torch.float32
            for r, s, want in zip(out.residuals, out.scale, down + [mid]):
                got = (r * s).reshape(want.shape[0], want.shape[2], want.shape[3], -1).permute(0, 3, 1, 2)
                assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


def test_scales_and_keep_formulas():
    from imagharmony_b200.controlnet import controlnet_keep, controlnet_scales
    assert torch.equal(controlnet_scales(0.8, False), torch.full((10,), 0.8))
    assert torch.equal(controlnet_scales(0.8, True), torch.logspace(-1, 0, 10) * 0.8)
    assert controlnet_scales(1.0, True)[-1] == 1.0 and abs(controlnet_scales(1.0, True)[0] - 0.1) < 1e-7
    for T, start, end in ((10, 0.0, 1.0), (10, 0.2, 1.0), (10, 0.0, 0.55), (7, 0.3, 0.8)):
        want = [1.0 - float(i / T < start or (i + 1) / T > end) for i in range(T)]
        assert controlnet_keep(T, start, end) == want
    assert controlnet_keep(10, 0.2, 0.55) == [0, 0, 1, 1, 1, 0, 0, 0, 0, 0]


def test_state_dict_keys_are_diffusers_names():
    from controlnet_ref import ControlNetRef
    from imagharmony_b200.config import SDXL_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetModel
    with torch.device("meta"):
        native, ref = ControlNetModel(SDXL_CONTROLNET), ControlNetRef(SDXL_CONTROLNET)
    keys = set(native.state_dict())
    assert keys == set(ref.state_dict())
    for k in ("controlnet_cond_embedding.conv_in.weight", "controlnet_cond_embedding.blocks.5.bias",
              "controlnet_cond_embedding.conv_out.weight", "controlnet_down_blocks.8.weight", "controlnet_mid_block.bias",
              "down_blocks.2.attentions.1.transformer_blocks.9.attn2.to_k.weight", "mid_block.resnets.1.conv2.weight",
              "add_embedding.linear_1.weight", "conv_in.weight"):
        assert k in keys, k
    assert not any(k.startswith("up_blocks") or k.startswith("conv_out") for k in keys)
    assert native.state_dict()["controlnet_down_blocks.8.weight"].shape == (1280, 1280, 1, 1)
    assert len(native.attn_processors) == 2 * (2 * 2 + 2 * 10 + 10)      # attn1 + attn2 of 34 transformer blocks


def test_from_pretrained_round_trip(tmp_path, cnp):
    from safetensors.torch import save_file
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetModel
    native, _ = _cn_pair(TINY_CONTROLNET, 1)
    sd = {k: v.half().contiguous() for k, v in native.state_dict().items()}
    save_file(sd, str(tmp_path / "diffusion_pytorch_model.fp16.safetensors"))
    c = TINY_CONTROLNET
    meta = {"_class_name": "ControlNetModel", "block_out_channels": list(c.block_out_channels),
            "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
            "transformer_layers_per_block": [1, 1, 2], "attention_head_dim": [1, 2, 4],
            "cross_attention_dim": c.cross_attention_dim, "addition_time_embed_dim": c.addition_time_embed_dim,
            "projection_class_embeddings_input_dim": 6 * c.addition_time_embed_dim + c.pooled_embed_dim,
            "conditioning_embedding_out_channels": list(c.conditioning_embedding_out_channels),
            "controlnet_conditioning_channel_order": "rgb", "global_pool_conditions": False, "in_channels": 4}
    (tmp_path / "config.json").write_text(json.dumps(meta))
    m = ControlNetModel.from_pretrained(str(tmp_path), device="cpu")
    assert m.config.transformer_layers_per_block == c.transformer_layers_per_block
    assert m.config.pooled_embed_dim == c.pooled_embed_dim
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    meta["global_pool_conditions"] = True
    (tmp_path / "config.json").write_text(json.dumps(meta))
    with pytest.raises(IHError):
        ControlNetModel.from_pretrained(str(tmp_path), device="cpu")
    meta["global_pool_conditions"] = False
    (tmp_path / "config.json").write_text(json.dumps(meta))
    save_file({k: v for k, v in sd.items() if k != "controlnet_mid_block.bias"},
              str(tmp_path / "diffusion_pytorch_model.fp16.safetensors"))
    with pytest.raises(RuntimeError):                  # strict keys
        ControlNetModel.from_pretrained(str(tmp_path), device="cpu")


def test_refusals():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetModel
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    with pytest.raises(IHError, match="global_pool"), torch.device("meta"):
        ControlNetModel(dataclasses.replace(TINY_CONTROLNET, global_pool_conditions=True))
    with pytest.raises(IHError, match="Multi-ControlNet"):
        StableDiffusionXLControlNetPipeline(None, [None, None])


def test_control_image_preprocessing():
    """[3P] VaeImageProcessor(do_normalize=False): Lanczos resize, [0, 1]; size from the image floored to 8."""
    from PIL import Image
    from ip_adapter.custom_pipelines import preprocess_control_image
    rng = np.random.default_rng(0)
    im = Image.fromarray(rng.integers(0, 256, (70, 83, 3), dtype=np.uint8))
    x = preprocess_control_image(im)
    want = np.array(im.resize((80, 64), resample=Image.LANCZOS)).astype(np.float32) / 255.0
    assert x.shape == (1, 3, 64, 80) and torch.equal(x, torch.from_numpy(want).permute(2, 0, 1)[None])
    x = preprocess_control_image([im, im], 32, 48)
    assert x.shape == (2, 3, 32, 48) and 0.0 <= x.min() and x.max() <= 1.0
    t = torch.rand(1, 3, 40, 40)
    assert torch.equal(preprocess_control_image(t), t)
    assert preprocess_control_image(t, 16, 24).shape == (1, 3, 16, 24)


def _pipe(cfg_cn=None, seed=0):
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    pipe = StableDiffusionXLControlNetPipeline.from_random(TINY, cfg_cn or TINY_CONTROLNET, seed=seed, device="cpu")
    for m in (pipe.unet, pipe.controlnet):
        m.float()
        m.finalize()
    return pipe


@pytest.mark.parametrize("opts", [dict(), dict(guess_mode=True, controlnet_conditioning_scale=0.6),
                                  dict(control_guidance_start=0.25, control_guidance_end=0.75),
                                  dict(guidance_scale=1.0, guess_mode=True)])
def test_pipeline_loop_matches_reference(cnp, opts):
    """StableDiffusionXLControlNetPipeline (engine eager steps, fp32 stand-in ops) against the restated diffusers loop:
    CFG, guess mode (the ControlNet on the conditional half), a keep window, no CFG; the generator is read only for
    the initial latents."""
    from controlnet_ref import ControlNetRef, UNetResidualRef, controlnet_denoise_loop
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from oracle import adapter_ref as A
    pipe = _pipe()
    ref_u = UNetResidualRef(TINY)
    A.install_processors(ref_u, TINY)
    ref_u.load_state_dict({k: v.float() for k, v in pipe.unet.state_dict().items()})
    torch.nn.ModuleList(p for p in ref_u.attn_processors.values() if hasattr(p, "to_k_ip")).load_state_dict(
        {k: v.float() for k, v in torch.nn.ModuleList(
            p for p in pipe.unet.attn_processors.values() if hasattr(p, "to_k_ip")).state_dict().items()})
    ref_c = ControlNetRef(TINY_CONTROLNET)
    ref_c.load_state_dict({k: v.float() for k, v in pipe.controlnet.state_dict().items()})
    ref_c.set_attn_processor({k: A.SelfAttnProcessorRef() for k in ref_c.attn_processors})
    n, lat, T = 1, 8, 4
    g = torch.Generator().manual_seed(7)
    pos, neg = torch.randn(n, 77, 128, generator=g), torch.randn(n, 77, 128, generator=g)
    pp, npool = torch.randn(n, 64, generator=g), torch.randn(n, 64, generator=g)
    img = _image(1, 8 * lat)
    gen = torch.Generator().manual_seed(11)
    kw = dict(guidance_scale=5.0, controlnet_conditioning_scale=1.0)
    kw.update(opts)
    with _Empty32():
        pipe.engine.use_cuda_graph = False
        out = pipe(prompt_embeds=pos, negative_prompt_embeds=neg, pooled_prompt_embeds=pp,
                   negative_pooled_prompt_embeds=npool, image=img, num_inference_steps=T, generator=gen,
                   output_type="latent", **kw).images
    assert torch.equal(gen.get_state(), _after_latents(n, lat))          # the ControlNet draws nothing
    from oracle.scheduler_ref import euler_tables
    _, _, ins = euler_tables(T)
    lat0 = torch.randn((n, 4, lat, lat), generator=torch.Generator().manual_seed(11)) * ins
    tid = torch.tensor([[8. * lat, 8. * lat, 0., 0., 8. * lat, 8. * lat]])
    with torch.no_grad():
        want = controlnet_denoise_loop(
            ref_u, ref_c, lat0, pos, neg, pp, npool, tid, img, T, guidance_scale=kw["guidance_scale"],
            conditioning_scale=kw["controlnet_conditioning_scale"], guess_mode=kw.get("guess_mode", False),
            control_guidance_start=kw.get("control_guidance_start", 0.0),
            control_guidance_end=kw.get("control_guidance_end", 1.0))
    assert torch.allclose(out.float(), want, rtol=1e-3, atol=1e-3), (out.float() - want).abs().max()


def _after_latents(n, lat):
    g = torch.Generator().manual_seed(11)
    torch.randn((n, 4, lat, lat), generator=g)
    return g.get_state()


def test_ip_adapter_installs_cn_processors_text_only(cnp):
    """IPAdapterXL on a ControlNet pipeline: CNAttnProcessor2_0 on every ControlNet attention; the ControlNet's
    cross-attention K/V are computed from the 77 text tokens only."""
    from imagharmony_b200.config import TINY
    from ip_adapter.attention_processor import CNAttnProcessor, CNAttnProcessor2_0
    from ip_adapter.ip_adapter import IPAdapterXL
    assert CNAttnProcessor is CNAttnProcessor2_0
    pipe = _pipe()
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    assert not hasattr(StableDiffusionXLCustomPipeline.from_random(TINY, device="cpu"), "controlnet")
    epoch = pipe.controlnet.graph_epoch
    ip = IPAdapterXL(pipe, None, None, "cpu", num_tokens=4)
    procs = list(pipe.controlnet.attn_processors.values())
    assert procs and all(isinstance(p, CNAttnProcessor2_0) and p.num_tokens == 4 for p in procs)
    assert pipe.controlnet.graph_epoch > epoch
    g = torch.Generator().manual_seed(1)
    ehs = torch.randn(2, 81, TINY.cross_attention_dim, generator=g)
    te, tid = torch.randn(2, TINY.pooled_embed_dim, generator=g), torch.tensor([[64., 64, 0, 0, 64, 64]] * 2)
    pipe.controlnet.float()
    pipe.controlnet.finalize()
    pipe.controlnet.prepare_conditioning(ehs, te, tid)
    p = procs[0]
    for name, attn in pipe.controlnet._attn_modules():
        if attn.is_cross:
            _, kv, nk, n_ip = p._text[id(attn)]._kv
            assert n_ip == 0
            assert nk == 77 and kv.shape[0] == 2 * 77
            want = ehs[:, :77].reshape(-1, ehs.shape[-1]) @ attn.fused_kv_weight().float().t()
            assert torch.allclose(kv.float(), want, atol=2e-3, rtol=2e-3)   # fp16 K/V buffer
    assert ip.pipe is pipe


@pytest.mark.parametrize("n_img, per_prompt, guess", [(1, 1, False), (1, 3, False), (2, 2, True)])
def test_control_image_batch_expansion(n_img, per_prompt, guess, monkeypatch):
    """[3P] prepare_image: one image is repeat_interleaved to the whole batch, a batch of images by
    num_images_per_prompt; the engine receives one image per latent (it duplicates the embedding for CFG unless guess
    mode).  Two prompts, so the batch is 2 * num_images_per_prompt."""
    from imagharmony_b200.controlnet import controlnet_keep
    pipe = _pipe()
    seen = {}

    def run(lat, *a, controlnet=None, **k):
        seen["cn"], seen["n"] = controlnet, lat.shape[0]
        return lat
    monkeypatch.setattr(pipe.engine, "run", run)
    imgs = _image(n_img if n_img > 1 else 1, 64)
    if n_img > 1:                                      # one control image per prompt
        imgs = torch.stack([imgs[0], _image(1, 64, seed=9)[0]])
    pipe(prompt=["a", "b"], image=imgs, num_images_per_prompt=per_prompt, num_inference_steps=5,
         output_type="latent", guess_mode=guess, controlnet_conditioning_scale=0.3, control_guidance_end=0.6)
    cn = seen["cn"]
    want = imgs.repeat_interleave(2 * per_prompt if n_img == 1 else per_prompt, dim=0).half()
    assert seen["n"] == 2 * per_prompt and torch.equal(cn.image, want)
    assert cn.guess_mode == guess and cn.conditioning_scale == 0.3 and cn.keep == controlnet_keep(5, 0.0, 0.6)
