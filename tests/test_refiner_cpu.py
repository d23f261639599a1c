"""CPU tests of the SDXL refiner and the base -> refiner handoff (ensemble of experts): the diffusers config parser, the
refiner architecture against the oracle (tests/refiner_ref.py) on the plain-PyTorch stand-in ops, the
denoising_start -> begin_step rule, the latent hand-over, the aesthetic-score time ids, single-tower prompt encoding,
and the two-pipeline ensemble against one restated loop that switches the model."""
import json

import pytest
import torch

from refiner_ref import begin_step_ref, ensemble_loop, unet_ref
from test_wiring_cpu import patched  # noqa: F401  (fixture)

REFINER_UNET_JSON = {
    "_class_name": "UNet2DConditionModel", "act_fn": "silu", "addition_embed_type": "text_time",
    "addition_time_embed_dim": 256, "attention_head_dim": [6, 12, 24, 24], "block_out_channels": [384, 768, 1536, 1536],
    "center_input_sample": False, "class_embed_type": None, "cross_attention_dim": 1280,
    "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"],
    "downsample_padding": 1, "dual_cross_attention": False, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4,
    "layers_per_block": 2, "mid_block_scale_factor": 1, "mid_block_type": "UNetMidBlock2DCrossAttn", "norm_eps": 1e-05,
    "norm_num_groups": 32, "num_attention_heads": None, "num_class_embeds": None, "only_cross_attention": False,
    "out_channels": 4, "projection_class_embeddings_input_dim": 2560, "resnet_time_scale_shift": "default",
    "sample_size": 128, "time_cond_proj_dim": None, "time_embedding_type": "positional", "timestep_post_act": None,
    "transformer_layers_per_block": 4,
    "up_block_types": ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"],
    "upcast_attention": None, "use_linear_projection": True}
BASE_UNET_JSON = {
    **REFINER_UNET_JSON, "attention_head_dim": [5, 10, 20], "block_out_channels": [320, 640, 1280],
    "cross_attention_dim": 2048, "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
    "up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"],
    "projection_class_embeddings_input_dim": 2816, "transformer_layers_per_block": [1, 2, 10], "upcast_attention": False}
TINY_REFINER_UNET_JSON = {
    **REFINER_UNET_JSON, "attention_head_dim": [1, 2, 4, 4], "block_out_channels": [64, 128, 256, 256],
    "cross_attention_dim": 192, "addition_time_embed_dim": 32, "projection_class_embeddings_input_dim": 5 * 32 + 64,
    "transformer_layers_per_block": [1, 1, 2, 1], "sample_size": 32}


# ---------------------------------------------------------------------------------------------------------------------
# config parser
# ---------------------------------------------------------------------------------------------------------------------
def test_parser_reads_refiner_and_base():
    from imagharmony_b200.config import SDXL_BASE, SDXL_REFINER, TINY_REFINER, UNetConfig, config_from_diffusers
    assert config_from_diffusers(REFINER_UNET_JSON, UNetConfig, requires_aesthetics_score=True) == SDXL_REFINER
    assert config_from_diffusers(BASE_UNET_JSON, UNetConfig) == SDXL_BASE
    assert config_from_diffusers(TINY_REFINER_UNET_JSON, UNetConfig, True) == TINY_REFINER
    # 2560 = 5 * 256 + 1280 = 6 * 256 + 1024: only model_index.json's requires_aesthetics_score tells them apart
    six = config_from_diffusers(REFINER_UNET_JSON, UNetConfig, requires_aesthetics_score=False)
    assert (six.num_time_ids, six.pooled_embed_dim) == (6, 1024) and six != SDXL_REFINER
    assert (SDXL_REFINER.num_time_ids, SDXL_REFINER.pooled_embed_dim, SDXL_REFINER.add_embed_in) == (5, 1280, 2560)
    assert SDXL_REFINER.mid_depth == 4 and SDXL_BASE.mid_depth == 10 and SDXL_BASE.add_embed_in == 2816
    assert SDXL_REFINER.time_embed_dim == 1536


@pytest.mark.parametrize("change", [
    {"attention_head_dim": [6, 12, 24, 12]},                                       # a level 128 wide per head
    {"attention_head_dim": 8},                                                     # 48 / 96 / 192-wide heads
    {"up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D", "UpBlock2D"]},   # not mirrored
    {"down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "SimpleCrossAttnDownBlock2D", "DownBlock2D"]},
    {"use_linear_projection": False}, {"addition_embed_type": "text"}, {"class_embed_type": "timestep"},
    {"mid_block_type": "UNetMidBlock2DSimpleCrossAttn"}, {"transformer_layers_per_block": [[1, 2], 4, 4, 4]},
    {"layers_per_block": [2, 2, 2, 2]}, {"encoder_hid_dim": 1024}, {"time_cond_proj_dim": 256},
    {"resnet_time_scale_shift": "scale_shift"}, {"projection_class_embeddings_input_dim": 1000},
    {"conv_in_kernel": 1}, {"only_cross_attention": True},
])
def test_parser_refuses_what_the_native_unet_cannot_build(change):
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import UNetConfig, config_from_diffusers
    with pytest.raises(IHError):
        config_from_diffusers({**REFINER_UNET_JSON, **change}, UNetConfig, requires_aesthetics_score=True)


def test_refiner_state_dict_matches_oracle():
    from imagharmony_b200.config import SDXL_REFINER
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import shapes_of
    with torch.device("meta"):
        native, ref = UNet2DConditionModel(SDXL_REFINER), unet_ref(SDXL_REFINER)
    assert shapes_of(native) == shapes_of(ref)
    assert native.add_embedding.linear_1.weight.shape == (1536, 2560)
    assert len(native.mid_block.attentions[0].transformer_blocks) == 4
    assert sum(r.cout for r in native.modules() if type(r).__name__ == "ResnetBlock2D") == 24192   # temb_all columns
    names = list(native.attn_processors)
    assert len(names) == 2 * (2 * 4 + 2 * 4 + 3 * 4 + 3 * 4 + 4) and "down_blocks.2.attentions.1.transformer_blocks.0.attn2.processor" in names


def test_refiner_processors_are_text_only():
    from imagharmony_b200.config import TINY_REFINER
    from imagharmony_b200.unet import UNet2DConditionModel
    from ip_adapter.attention_processor import CNAttnProcessor2_0
    with torch.device("meta"):
        m = UNet2DConditionModel(TINY_REFINER)
    m.install_default_processors()
    procs = set(map(id, m.attn_processors.values()))
    assert len(procs) == 1
    p = next(iter(m.attn_processors.values()))
    assert isinstance(p, CNAttnProcessor2_0) and p.num_tokens == 0 and not hasattr(p, "to_k_ip")


# ---------------------------------------------------------------------------------------------------------------------
# wiring of the refiner on the stand-in ops
# ---------------------------------------------------------------------------------------------------------------------
def _pair(cfg, seed):
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(unet_ref(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, seed).items()}
    with torch.device("meta"):
        native = UNet2DConditionModel(cfg)
    native.load_state_dict(sd, assign=True)
    native.install_default_processors()
    native.finalize()
    ref = unet_ref(cfg)
    ref.load_state_dict(sd)
    return native, ref.eval()


def _record_attention(monkeypatch):
    import imagharmony_b200.ops as real_ops
    seen, inner = [], real_ops.attention

    def attention(q, k, v, B, H, Nq, Nk, **kw):
        seen.append((H, Nq, Nk, kw.get("n_ip", 0)))
        return inner(q, k, v, B, H, Nq, Nk, **kw)
    monkeypatch.setattr(real_ops, "attention", attention)
    return seen


def test_tiny_refiner_wiring_matches_oracle(patched, monkeypatch):  # noqa: F811
    from imagharmony_b200.config import TINY_REFINER as cfg
    native, ref = _pair(cfg, 0)
    seen = _record_attention(monkeypatch)
    g = torch.Generator().manual_seed(1)
    B, lat = 2, 16
    sample = torch.randn(B, 4, lat, lat, generator=g)
    ehs = torch.randn(B, 77, cfg.cross_attention_dim, generator=g)
    te = torch.randn(B, cfg.pooled_embed_dim, generator=g)
    tid = torch.tensor([[128., 128., 0., 0., 2.5], [128., 128., 0., 0., 6.0]])
    with torch.no_grad():
        r = ref(sample, 321.0, ehs, te, tid)
        o = native(sample, torch.full((B,), 321.0), ehs, te, tid)
    assert o.shape == r.shape and torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()
    assert list(native.attn_processors) == list(ref.attn_processors)
    cross = [s for s in seen if s[2] != s[1]]
    assert cross and all(s[2] == 77 and s[3] == 0 for s in cross) and all(s[3] == 0 for s in seen)
    # the aesthetic score is conditioning: another score changes the output
    with torch.no_grad():
        o2 = native(sample, torch.full((B,), 321.0), ehs, te, tid.clone().fill_(3.0))
    assert (o2 - o).abs().max() > 1e-3
    from imagharmony_b200._lib import IHError
    with pytest.raises(IHError):                                     # 6 ids on a 5-id UNet
        native(sample, torch.full((B,), 321.0), ehs, te, torch.zeros(B, 6))


def test_refiner_needs_64_pixel_multiples():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import SDXL_BASE, SDXL_REFINER
    from imagharmony_b200.unet import require_latent_size
    from test_unet_census_gpu import BUCKETS
    for h, w in BUCKETS:
        require_latent_size(SDXL_REFINER, h // 8, w // 8)
    require_latent_size(SDXL_BASE, 132, 128)
    with pytest.raises(IHError):
        require_latent_size(SDXL_REFINER, 132, 128)                  # 1056 x 1024


# ---------------------------------------------------------------------------------------------------------------------
# pipelines
# ---------------------------------------------------------------------------------------------------------------------
def _refiner_pipe(**kw):
    from imagharmony_b200.config import TINY_REFINER
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    return StableDiffusionXLImg2ImgPipeline.from_random(TINY_REFINER, seed=3, device="cpu", **kw)


class _Runs:
    """DenoiseEngine.run replaced by a recorder that returns its input latents."""

    def __init__(self, monkeypatch):
        from imagharmony_b200.denoise import DenoiseEngine
        self.calls = []

        def run(engine, latents, *a, **k):
            self.calls.append((latents.clone(), a, k))
            return latents.clone()
        monkeypatch.setattr(DenoiseEngine, "run", run)


def test_begin_step_matches_get_timesteps_and_base_loop_end(monkeypatch):
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline, denoising_start_begin_step
    from imagharmony_b200.config import TINY
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    from oracle.scheduler_ref import denoising_end_steps
    fractions = [0.01, 0.05, 0.1, 0.2, 0.25, 0.3, 1 / 3, 0.5, 0.6, 0.7, 0.75, 0.8, 0.9, 0.95, 0.999]
    sched = EulerDiscreteScheduler()
    for T in range(1, 101):
        sched.set_timesteps(T)
        for d in fractions:
            b = denoising_start_begin_step(sched.timesteps, sched.num_train_timesteps, d)
            assert b == begin_step_ref(T, d) == denoising_end_steps(T, d), (T, d)
    for bad in (0.0, 1.0, 1.5, -0.2, 1, "0.5", None):
        assert begin_step_ref(10, bad) is None
    # through the pipelines: the base's loop end and the refiner's begin step for the same fraction
    runs = _Runs(monkeypatch)
    base, ref = StableDiffusionXLCustomPipeline.from_random(TINY, device="cpu"), _refiner_pipe()
    lat = torch.zeros(1, 4, 8, 8, dtype=torch.float16)
    for T, d in ((10, 0.8), (50, 0.5), (3, 0.05), (3, 0.999)):      # the last two: the base / the refiner runs no step
        if True:
            runs.calls.clear()
            base(prompt="a", num_inference_steps=T, denoising_end=d, output_type="latent", height=64, width=64)
            ends = [c[2]["num_loop_steps"] for c in runs.calls]
            runs.calls.clear()
            ref(prompt="a", image=lat, num_inference_steps=T, denoising_start=d, output_type="latent")
            begins = [c[2]["begin_step"] for c in runs.calls]
            want = begin_step_ref(T, d)
            assert ends == ([want] if want > 0 else []), (T, d, ends)
            assert begins == ([want] if want < T else []), (T, d, begins)


def test_latent_image_reaches_the_engine_unchanged(monkeypatch):
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    pipe = _refiner_pipe(vae_cfg=TINY_VAE)
    pipe.scheduler = EulerAncestralDiscreteScheduler()

    def no_vae(*a, **k):
        raise AssertionError("the hand-over latents must not be encoded")
    monkeypatch.setattr(pipe.vae_encoder, "encode_moments_nhwc", no_vae)
    runs = _Runs(monkeypatch)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(2)).half()
    g = torch.Generator().manual_seed(5)
    state = g.get_state()
    out = pipe(prompt="lions", image=lat, num_inference_steps=10, denoising_start=0.8, num_images_per_prompt=2,
               generator=g, output_type="latent").images
    (got, args, kw), = runs.calls
    assert torch.equal(got, lat.repeat(2, 1, 1, 1)) and got.dtype == torch.float16
    assert kw["begin_step"] == begin_step_ref(10, 0.8) == 8 and args[5] == 10 and kw["generator"] is g
    assert torch.equal(g.get_state(), state)                          # no draw in the pipeline
    assert torch.equal(out, got)
    # n = 0: the input latents come back, the engine does not run
    runs.calls.clear()
    out = pipe(prompt="lions", image=lat, num_inference_steps=10, denoising_start=0.999, output_type="latent").images
    assert not runs.calls and torch.equal(out, lat)


def test_aesthetic_time_ids(monkeypatch):
    pipe = _refiner_pipe()
    runs = _Runs(monkeypatch)
    lat = torch.zeros(1, 4, 8, 8, dtype=torch.float16)
    pipe(prompt="a", image=lat, num_inference_steps=10, denoising_start=0.5, output_type="latent")
    _, args, kw = runs.calls[-1]
    assert args[4].tolist() == [[64.0, 64.0, 0.0, 0.0, 6.0]] and kw["negative_time_ids"].tolist() == [[64.0, 64.0, 0.0, 0.0, 2.5]]
    pipe(prompt="a", image=lat, num_inference_steps=10, denoising_start=0.5, output_type="latent", num_images_per_prompt=2,
         original_size=(1024, 768), crops_coords_top_left=(3, 4), target_size=(9, 9), aesthetic_score=7.0,
         negative_aesthetic_score=1.5, negative_original_size=(512, 384), negative_crops_coords_top_left=(1, 2))
    _, args, kw = runs.calls[-1]
    assert args[4].tolist() == [[1024.0, 768.0, 3.0, 4.0, 7.0]] * 2
    assert kw["negative_time_ids"].tolist() == [[512.0, 384.0, 1.0, 2.0, 1.5]] * 2


def test_refusals():
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_CONTROLNET, TINY_VAE
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import (StableDiffusionXLControlNetPipeline, StableDiffusionXLCustomPipeline,
                                             StableDiffusionXLInpaintPipeline)
    pipe = _refiner_pipe(vae_cfg=TINY_VAE)
    lat = torch.zeros(1, 4, 8, 8, dtype=torch.float16)
    common = dict(prompt="a", num_inference_steps=10, output_type="latent")
    for cls in (StableDiffusionXLCustomPipeline, StableDiffusionXLInpaintPipeline):
        with pytest.raises(IHError):
            cls(pipe.unet)
    from imagharmony_b200.controlnet import ControlNetModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(ControlNetModel(TINY_CONTROLNET))
    with pytest.raises(IHError):
        StableDiffusionXLControlNetPipeline(pipe.unet, ControlNetModel.from_state_dict(
            TINY_CONTROLNET, random_state_dict(shapes, 1), device="cpu"))
    with pytest.raises(IHError):
        IPAdapterXL(pipe, None, None, "cpu", num_tokens=4)
    with pytest.raises(ValueError):
        pipe(image=lat, denoising_start=0.8, denoising_end=0.8, **common)
    with pytest.raises(ValueError):
        pipe(image=lat, denoising_start=0.8, strength=1.5, **common)
    with pytest.raises(IHError):                                     # latents need a valid denoising_start
        pipe(image=lat, **common)
    with pytest.raises(IHError):
        pipe(image=lat, denoising_start=1.0, **common)
    with pytest.raises(IHError):                                     # 1056 x 1024: not a multiple of 64 px
        pipe(image=torch.zeros(1, 4, 132, 128, dtype=torch.float16), denoising_start=0.8, **common)
    pipe.scheduler = DPMSolverMultistepScheduler()
    with pytest.raises(IHError):
        pipe(image=lat, denoising_start=0.8, **common)


def test_invalid_denoising_start_is_ignored(patched, monkeypatch):  # noqa: F811
    """A denoising_start that is not a float in (0, 1) is ignored, as in diffusers: plain image-to-image."""
    import fake_ops_img2img
    import imagharmony_b200.ops as real_ops
    from imagharmony_b200.config import TINY, TINY_VAE
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    for name in fake_ops_img2img.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_img2img, name))
    pipe = StableDiffusionXLImg2ImgPipeline.from_random(TINY, device="cpu", vae_cfg=TINY_VAE)
    init = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(0)) * 2 - 1
    outs = [pipe(prompt="a", image=init, strength=0.5, num_inference_steps=4, output_type="latent",
                 generator=torch.Generator().manual_seed(1), **kw).images for kw in ({}, {"denoising_start": 1.5},
                                                                                    {"denoising_start": 1})]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ---------------------------------------------------------------------------------------------------------------------
# prompt encoding and loading
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def clip_ops(monkeypatch):
    import fake_ops
    import imagharmony_b200.clip as clip
    import imagharmony_b200.ops as real_ops
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real_ops, name):
            monkeypatch.setattr(real_ops, name, getattr(fake_ops, name))
    monkeypatch.setattr(clip, "_DTYPE", [torch.float32])
    yield


def test_single_tower_prompt_encoding(tmp_path, clip_ops):
    pytest.importorskip("transformers")
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    from test_encoders_cpu import _toy_tokenizer
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    from ip_adapter.encoders import ClipPromptEncoder
    tok2, nv = _toy_tokenizer(tmp_path, "t2")
    torch.manual_seed(0)
    e2 = CLIPTextModelWithProjection(CLIPTextConfig(
        hidden_size=48, intermediate_size=96, projection_dim=40, vocab_size=nv, max_position_embeddings=77,
        num_hidden_layers=3, num_attention_heads=2, bos_token_id=nv - 2, eos_token_id=nv - 1, pad_token_id=nv - 1))
    enc = ClipPromptEncoder(None, tok2, None, e2, device="cpu", dtype=torch.float32)
    prompts = ["eight sheep", ""]
    hs, pooled = enc(prompts)
    with torch.no_grad():
        ids = tok2(prompts, padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
        o = e2(ids, output_hidden_states=True)
    assert hs.shape == (2, 77, 48) and pooled.shape == (2, 40)
    assert torch.allclose(hs.float(), o.hidden_states[-2], atol=2e-3)
    assert torch.allclose(pooled.float(), o.text_embeds, atol=2e-3)
    with pytest.raises(ValueError):
        ClipPromptEncoder(tok2, tok2, None, e2, device="cpu")
    # force_zeros_for_empty_prompt = false (the refiner's model_index.json): no negative prompt -> "" encoded
    pipe = _refiner_pipe()
    pipe.prompt_encoder = enc
    pipe._configure({"force_zeros_for_empty_prompt": False})
    pe, ne, pp, npool = pipe.encode_prompt("eight sheep", num_images_per_prompt=2)
    want_ne, want_np = enc([""])
    assert torch.equal(ne, want_ne.repeat(2, 1, 1)) and torch.equal(npool, want_np.repeat(2, 1))
    assert torch.count_nonzero(ne) > 0
    assert StableDiffusionXLImg2ImgPipeline.force_zeros_for_empty_prompt is True      # per instance, base default


def test_from_pretrained_reads_the_refiner_folder(tmp_path):
    from safetensors.torch import save_file
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY_REFINER
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline, StableDiffusionXLImg2ImgPipeline
    from ip_adapter.encoders import ClipPromptEncoder
    with torch.device("meta"):
        shapes = shapes_of(UNet2DConditionModel(TINY_REFINER))
    (tmp_path / "unet").mkdir()
    save_file(random_state_dict(shapes, 4), str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
    (tmp_path / "unet" / "config.json").write_text(json.dumps(TINY_REFINER_UNET_JSON))
    (tmp_path / "model_index.json").write_text(json.dumps({"_class_name": "StableDiffusionXLImg2ImgPipeline",
                                                           "requires_aesthetics_score": True,
                                                           "force_zeros_for_empty_prompt": False}))
    pipe = StableDiffusionXLImg2ImgPipeline.from_pretrained(str(tmp_path), device="cpu")
    assert pipe.unet.config == TINY_REFINER and pipe.force_zeros_for_empty_prompt is False
    with pytest.raises(IHError):
        StableDiffusionXLCustomPipeline.from_pretrained(str(tmp_path), device="cpu")
    for d in ("tokenizer_2", "text_encoder_2"):
        (tmp_path / d).mkdir()
    assert ClipPromptEncoder.available(str(tmp_path))


# ---------------------------------------------------------------------------------------------------------------------
# the ensemble: base to k, refiner from k
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ancestral", [False, True], ids=["euler", "euler_a"])
def test_ensemble_matches_restated_switching_loop(patched, monkeypatch, ancestral):  # noqa: F811
    import fake_ops_euler_a
    import imagharmony_b200.ops as real_ops
    for name in fake_ops_euler_a.NAMES:
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_euler_a, name))
    from imagharmony_b200.config import TINY, TINY_REFINER
    from imagharmony_b200.scheduler import EulerAncestralDiscreteScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    from oracle import adapter_ref as A
    from oracle.scheduler_ref import euler_tables
    from oracle.unet_ref import UNetRef
    T, d, gs = 5, 0.6, 5.0
    k = begin_step_ref(T, d)
    assert 0 < k < T
    base, refiner = StableDiffusionXLCustomPipeline.from_random(TINY, seed=1, device="cpu"), _refiner_pipe()
    if ancestral:
        base.scheduler, refiner.scheduler = EulerAncestralDiscreteScheduler(), EulerAncestralDiscreteScheduler()
    g = torch.Generator().manual_seed(9)
    emb = torch.Generator().manual_seed(4)
    b_pe, b_ne = (torch.randn(1, 77 + TINY.num_ip_tokens, TINY.cross_attention_dim, generator=emb).half() for _ in "ab")
    b_pp, b_np = (torch.randn(1, TINY.pooled_embed_dim, generator=emb).half() for _ in "ab")
    r_pe, r_ne = (torch.randn(1, 77, TINY_REFINER.cross_attention_dim, generator=emb).half() for _ in "ab")
    r_pp, r_np = (torch.randn(1, TINY_REFINER.pooled_embed_dim, generator=emb).half() for _ in "ab")
    mid = base(prompt_embeds=b_pe, negative_prompt_embeds=b_ne, pooled_prompt_embeds=b_pp,
               negative_pooled_prompt_embeds=b_np, num_inference_steps=T, denoising_end=d, guidance_scale=gs,
               height=64, width=64, generator=g, output_type="latent").images
    out = refiner(prompt_embeds=r_pe, negative_prompt_embeds=r_ne, pooled_prompt_embeds=r_pp,
                  negative_pooled_prompt_embeds=r_np, image=mid, num_inference_steps=T, denoising_start=d,
                  guidance_scale=gs, generator=g, output_type="latent").images

    ref_b = UNetRef(TINY)
    ref_b.load_state_dict({k_: v.float() for k_, v in base.unet.state_dict().items() if ".processor." not in k_})
    procs = A.install_processors(ref_b, TINY)
    torch.nn.ModuleList(procs.values()).load_state_dict(
        {k_: v.float() for k_, v in torch.nn.ModuleList(base.unet.attn_processors.values()).state_dict().items()})
    ref_r = unet_ref(TINY_REFINER)
    ref_r.load_state_dict({k_: v.float() for k_, v in refiner.unet.state_dict().items()})
    g2 = torch.Generator().manual_seed(9)
    _, _, ins = euler_tables(T)
    lat0 = (torch.randn((1, 4, 8, 8), generator=g2, dtype=torch.float32) * ins).half().float()
    tid_b = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    tid_r = torch.tensor([[64.0, 64.0, 0.0, 0.0, 2.5], [64.0, 64.0, 0.0, 0.0, 6.0]])
    cond_b = (torch.cat([b_ne, b_pe]).float(), torch.cat([b_np, b_pp]).float(), tid_b)
    cond_r = (torch.cat([r_ne, r_pe]).float(), torch.cat([r_np, r_pp]).float(), tid_r)
    want = ensemble_loop(lambda s, t, e, x, y: ref_b(s, t, e, x, y), cond_b,
                         lambda s, t, e, x, y: ref_r(s, t, e, x, y), cond_r, k, lat0, T, gs, ancestral, g2)
    err, mx = (out.float() - want.float()).abs().max().item(), want.float().abs().max().item()
    assert out.shape == (1, 4, 8, 8) and err <= 2e-2 * mx, (err, mx)
    if ancestral:       # the two pipelines drew from the generator exactly what the one loop draws, in its order
        assert torch.equal(g.get_state(), g2.get_state())
    if not ancestral:   # switching one step later gives another result
        off = ensemble_loop(lambda s, t, e, x, y: ref_b(s, t, e, x, y), cond_b,
                            lambda s, t, e, x, y: ref_r(s, t, e, x, y), cond_r, k + 1, lat0, T, gs)
        assert (off.float() - want.float()).abs().max() > 10 * err
