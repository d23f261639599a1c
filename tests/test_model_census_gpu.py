"""Per-call census (tests/census.py) of every model the product runs besides the UNet with n_ip = 4 and the untiled VAE
decoder (those are test_unet_census_gpu.py), at the sizes they are used at:

* the SDXL VAE encoder at every SDXL bucket plus 512^2 and 768^2, and its moments through the img2img posterior +
  add_noise kernel for 1 and 4 noise draws of one image;
* the VAE decoder and encoder with `use_tiling` (pipeline.enable_vae_tiling) at the eight buckets with a side over
  1024 px: their ragged edge tiles (decode 1216 x 832: latent tiles 128x104, 128x8, 56x104, 56x8; encode: image tiles
  1024x832, 1024x64, 448x832, 448x64);
* the SDXL ControlNet (conditioning embedding at the full image resolution, then the net) and the SDXL-base UNet with
  its residuals injected, at every bucket, 2 and 4 images, guess mode and without CFG; Multi-ControlNet with 2 and 3
  nets;
* the 9-channel inpainting UNet at every bucket;
* both SDXL CLIP text towers at batch 1, 2 and 8, the ViT-bigG vision tower at batch 1 and 4, and the PNS judge's
  resize of decoded candidates to 224^2;
* the tiny autoencoder decoder (TAESD-XL) at every bucket, batch 1, and at 1024^2 and 832 x 1216 with 4 and 8 images:
  its ReLU epilogue on conv_in's GEMM and on every block conv, and conv_out at alpha = 2 with Cout padded to 16;
* ImageProjModel, HarmonyAttention and the IP-Adapter Plus Resampler (also with its position-embedding and mean-pooled
  latent options) at batch 1, 2 and 4, and the SDXL UNet with the 16-token processors of IPAdapterPlusXL.

Random weights, eager forwards; the first call of each distinct key is checked (every call of the tiny decoder at
1024^2, one image).  `-s` prints one row per key and, at the end, how many keys each op got next to the coverage
summary of the UNet census."""
import dataclasses
import time
import types
import zlib

import pytest
import torch

import census
from test_kernels_gpu import ops  # noqa: F401  (fixture: TF32 off for the fp32 references)
from test_unet_census_gpu import BUCKETS, COVERED, _finish, plan

pytestmark = pytest.mark.gpu

TILED = [(h, w) for h, w in BUCKETS if max(h, w) > 1024]
OP_KEYS = {}


@pytest.fixture(scope="module", autouse=True)
def keys_per_op():
    yield
    print("\n== census coverage: " + ", ".join(f"{len(v)} {k}" for k, v in COVERED.items()))
    print("== census keys per op: " + ", ".join(f"{op} {len(k)}" for op, k in sorted(OP_KEYS.items())))


def _done(c, title):
    for key, r in c.rows.items():
        OP_KEYS.setdefault(r["op"], set()).add(key)
    _finish(c, title)


def _gen(*seed):
    return torch.Generator("cpu").manual_seed(zlib.crc32(repr(seed).encode()))


def _sdxl_unet(cfg):
    import bench
    return bench.build_native(cfg, "cuda")


def _conditioning(cfg, B, height, width, g):
    ehs = torch.randn(B, 77 + cfg.num_ip_tokens, cfg.cross_attention_dim, generator=g).half().cuda()
    te = torch.randn(B, cfg.pooled_embed_dim, generator=g).half().cuda()
    tid = torch.tensor([[height, width, 0., 0., height, width]] * B, device="cuda")
    return ehs, te, tid


# ---------------------------------------------------------------------------------------------------------------------
# VAE encoder (untiled and tiled) and tiled decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sdxl_vae_encoder(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_VAE
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLEncoder(SDXL_VAE))
    return AutoencoderKLEncoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 3, device="cuda"), device="cuda")


@pytest.fixture(scope="module")
def sdxl_vae_decoder(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_VAE
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLDecoder(SDXL_VAE))
    return AutoencoderKLDecoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 2, device="cuda"), device="cuda")


def _image(n, height, width, g):
    return (torch.rand(n, 3, height, width, generator=g) * 2 - 1).half().cuda()


ENCODER_CASES = [(h, w, 1) for h, w in BUCKETS] + [(1024, 1024, 2)]


@pytest.mark.parametrize("height,width,n", ENCODER_CASES, ids=[f"{h}x{w}-n{n}" for h, w, n in ENCODER_CASES])
def test_vae_encoder_census(ops, sdxl_vae_encoder, monkeypatch, height, width, n):  # noqa: F811
    enc = sdxl_vae_encoder
    g = _gen("enc", height, width, n)
    img = _image(n, height, width, g)
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    moments = enc.encode_moments_nhwc(img)
    h, w = height // 8, width // 8
    # the img2img latent preparation: one image's moments for n = 1 and 4 noise draws, fp32 eps (the upcast VAE)
    eps = torch.randn(1, 4, h, w, generator=g).cuda()
    for draws in (1, 4):
        noise = torch.randn(draws, 4, h, w, generator=g).half().cuda()
        lat = ops.vae_posterior_noise(moments[:1].contiguous(), eps, noise, 4, enc.config.scaling_factor, 3.0742)
        assert lat.shape == (draws, 4, h, w)
    monkeypatch.undo()
    assert moments.shape == (n, h, w, enc.MOMENT_PAD)
    assert {"conv3x3_down", "vae_posterior_noise"} <= {r["op"] for r in c.rows.values()}
    _done(c, f"VAE encoder {height}x{width} n={n}")


def tile_shapes(h, w, tile, stride):
    """The tile sizes of the tiled VAE: a restatement of the grid of vae.py _tiled_decode / _tiled_encode (tiles of
    `tile` every `stride`, the last ones cut at the edge), which labels what the census must have seen."""
    return {(min(tile, h - i), min(tile, w - j)) for i in range(0, h, stride) for j in range(0, w, stride)}


@pytest.mark.parametrize("height,width", TILED, ids=[f"{h}x{w}" for h, w in TILED])
def test_vae_tiled_census(ops, sdxl_vae_decoder, sdxl_vae_encoder, monkeypatch, height, width):  # noqa: F811
    dec, enc = sdxl_vae_decoder, sdxl_vae_encoder
    cfg = dec.config
    g = _gen("tiled", height, width)
    z = torch.randn(1, 4, height // 8, width // 8, generator=g).half().cuda()
    img = _image(1, height, width, g)
    monkeypatch.setattr(dec, "use_tiling", True)
    monkeypatch.setattr(enc, "use_tiling", True)
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    out = dec.decode(z)
    moments = enc.encode_moments_nhwc(img)
    monkeypatch.undo()
    assert out.shape == (1, 3, height, width) and moments.shape[1:3] == (height // 8, width // 8)
    tl = cfg.tile_latent_min_size
    dec_tiles = tile_shapes(height // 8, width // 8, tl, int(tl * (1 - cfg.tile_overlap_factor)))
    ts = cfg.sample_size
    enc_tiles = tile_shapes(height, width, ts, int(ts * (1 - cfg.tile_overlap_factor)))
    seen = {r["shape"] for r in c.rows.values() if r["op"] == "im2col3x3_nchw"}
    assert {f"1x5x{a}x{b}" for a, b in dec_tiles} <= seen, (dec_tiles, seen)     # latents | the constant-one channel
    assert {f"1x3x{a}x{b}" for a, b in enc_tiles} <= seen, (enc_tiles, seen)
    if (height, width) in ((1216, 832), (832, 1216)):
        assert min(min(t) for t in dec_tiles) == 8 and min(min(t) for t in enc_tiles) == 64
    print(f"\n[tiles {height}x{width}] decode {sorted(dec_tiles)} encode {sorted(enc_tiles)}")
    _done(c, f"tiled VAE {height}x{width}")


# ---------------------------------------------------------------------------------------------------------------------
# tiny autoencoder decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def taesdxl(ops):  # noqa: F811
    from imagharmony_b200.config import TAESDXL
    from imagharmony_b200.taesd import AutoencoderTinyDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from taesd_ref import AutoencoderTinyRef
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderTinyRef(TAESDXL))
    return AutoencoderTinyDecoder.from_state_dict(TAESDXL, random_state_dict(shapes, 14, device="cuda"), device="cuda")


TAESD_CASES = [(h, w, 1) for h, w in BUCKETS] + [(h, w, n) for h, w in ((1024, 1024), (832, 1216)) for n in (4, 8)]


@pytest.mark.parametrize("height,width,n", TAESD_CASES, ids=[f"{h}x{w}-n{n}" for h, w, n in TAESD_CASES])
def test_taesd_census(ops, taesdxl, monkeypatch, height, width, n):  # noqa: F811
    g = _gen("taesd", height, width, n)
    z = (torch.randn(n, 4, height // 8, width // 8, generator=g) * 3).half().cuda()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    c = census.Census(ops, check_all=(height, width, n) == (1024, 1024, 1), plan=plan).install(monkeypatch)
    img = taesdxl.decode(z)
    monkeypatch.undo()
    torch.cuda.synchronize()
    print(f"\n[taesd census {height}x{width} n={n}] {time.perf_counter() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated")
    assert img.shape == (n, 3, height, width)
    flags = {(r["op"], f) for r in c.rows.values() for f in r["shape"].split()}
    assert {("linear", "relu"), ("conv3x3", "relu")} <= flags, "the ReLU epilogue must run on the GEMM and the conv"
    assert any(r["op"] == "conv3x3" and r["shape"].split("->")[1].startswith("16 ") and "alpha=2" in r["shape"]
               for r in c.rows.values()), "conv_out: Cout padded to 16, alpha = 2"
    del img, z
    _done(c, f"TAESD-XL decoder {height}x{width} n={n}")
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# ControlNet + UNet with injected residuals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sdxl_unet(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_BASE
    return _sdxl_unet(SDXL_BASE)


@pytest.fixture(scope="module")
def sdxl_controlnet(ops):  # noqa: F811
    from controlnet_ref import ControlNetRef
    from imagharmony_b200.config import SDXL_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(ControlNetRef(SDXL_CONTROLNET))
    return ControlNetModel.from_state_dict(SDXL_CONTROLNET, random_state_dict(shapes, 4, device="cuda"))


def _controlnet_call(ops, unet, net, height, width, n, cfg, guess, k, monkeypatch, check_all=False):  # noqa: F811
    B = 2 * n if cfg else n
    g = _gen("cn", height, width, n, cfg, guess, k)
    h, w = height // 8, width // 8
    sample = torch.randn(B, 4, h, w, generator=g).half().cuda()
    ehs, te, tid = _conditioning(unet.config, B, height, width, g)
    t = torch.full((B,), 501.0, device="cuda")
    rows = slice(n, 2 * n) if guess else slice(0, B)          # guess mode: the ControlNet sees the conditional half
    c = census.Census(ops, check_all=check_all, plan=plan).install(monkeypatch)
    with torch.no_grad():
        outs = []
        for j in range(k):
            image = torch.rand(rows.stop - rows.start, 3, height, width, generator=g).half().cuda()
            emb = net.embed_condition(image)
            outs.append(net(sample[rows], t[rows], ehs[rows, :77].contiguous(), cond_embedding=emb,
                            conditioning_scale=0.8 - 0.2 * j, guess_mode=guess, text_embeds=te[rows], time_ids=tid[rows]))
        out = unet(sample, t, ehs, te, tid, controlnet_residuals=(outs[0] if k == 1 else outs, rows.start))
    monkeypatch.undo()
    assert out.shape == (B, 4, h, w)
    inject = "controlnet_add_residuals" if k == 1 else "controlnet_add_residuals_multi"
    rows_seen = [r for r in c.rows.values() if r["op"] == inject]
    assert rows_seen and all(r["checked"] for r in rows_seen), f"{inject} did not run under the census"
    assert any(r["op"] == "conv3x3_small" and " nchw" in r["shape"] for r in c.rows.values())
    return c


CN_CASES = ([(h, w, 1, True, False) for h, w in BUCKETS] + [(1024, 1024, n, True, False) for n in (2, 4)]
            + [(832, 1216, n, True, False) for n in (2, 4)] + [(1024, 1024, 1, True, True), (1024, 1024, 1, False, False)])


@pytest.mark.parametrize("height,width,n,cfg,guess", CN_CASES,
                         ids=[f"{h}x{w}-n{n}{'' if c else '-nocfg'}{'-guess' if gm else ''}" for h, w, n, c, gm in CN_CASES])
def test_controlnet_census(ops, sdxl_unet, sdxl_controlnet, monkeypatch, height, width, n, cfg, guess):  # noqa: F811
    c = _controlnet_call(ops, sdxl_unet, sdxl_controlnet, height, width, n, cfg, guess, 1, monkeypatch,
                         check_all=(height, width, n, cfg, guess) == (1024, 1024, 1, True, False))
    _done(c, f"ControlNet + UNet {height}x{width} n={n} cfg={cfg} guess={guess}")


MULTI_CASES = [(2, 1024, 1024, False), (2, 1216, 832, False), (3, 1024, 1024, True)]


@pytest.mark.parametrize("k,height,width,guess", MULTI_CASES,
                         ids=[f"K{k}-{h}x{w}{'-guess' if gm else ''}" for k, h, w, gm in MULTI_CASES])
def test_multi_controlnet_census(ops, sdxl_unet, sdxl_controlnet, monkeypatch, k, height, width, guess):  # noqa: F811
    c = _controlnet_call(ops, sdxl_unet, sdxl_controlnet, height, width, 1, True, guess, k, monkeypatch)
    _done(c, f"Multi-ControlNet K={k} {height}x{width} guess={guess}")


# ---------------------------------------------------------------------------------------------------------------------
# 9-channel inpainting UNet
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sdxl_unet9(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_BASE
    return _sdxl_unet(dataclasses.replace(SDXL_BASE, in_channels=9))


INPAINT_CASES = [(h, w, 1) for h, w in BUCKETS] + [(1024, 1024, 2)]


@pytest.mark.parametrize("height,width,n", INPAINT_CASES, ids=[f"{h}x{w}-n{n}" for h, w, n in INPAINT_CASES])
def test_unet9_census(ops, sdxl_unet9, monkeypatch, height, width, n):  # noqa: F811
    unet = sdxl_unet9
    B = 2 * n
    g = _gen("unet9", height, width, n)
    h, w = height // 8, width // 8
    sample = torch.randn(B, 4, h, w, generator=g).half().cuda()
    cond = torch.cat([(torch.rand(B, 1, h, w, generator=g) > 0.5).float(), torch.randn(B, 4, h, w, generator=g)], 1)
    ehs, te, tid = _conditioning(unet.config, B, height, width, g)
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    with torch.no_grad():
        out = unet(sample, torch.full((B,), 501.0, device="cuda"), ehs, te, tid, cond=cond.half().cuda())
    monkeypatch.undo()
    assert out.shape == (B, 4, h, w)
    assert any(r["op"] == "im2col3x3_nchw_cat" for r in c.rows.values())
    _done(c, f"9-channel UNet {height}x{width} n={n}")


# ---------------------------------------------------------------------------------------------------------------------
# CLIP towers and the PNS judge's resize
# ---------------------------------------------------------------------------------------------------------------------
def _hf_meta(cls_name, config_name, **kw):
    transformers = pytest.importorskip("transformers")
    with torch.device("meta"):
        return getattr(transformers, cls_name)(getattr(transformers, config_name)(**kw))


def _tower(cls, hf, seed):
    """A native tower with random weights in the layout of the (meta-device) transformers model `hf`."""
    from imagharmony_b200.clip import ClipTowerConfig
    from imagharmony_b200.weights import random_state_dict, shapes_of
    shapes = {k: s for k, s in shapes_of(hf).items() if not k.endswith("position_ids")}
    return cls(ClipTowerConfig.from_hf(hf.config), random_state_dict(shapes, seed), device="cuda")


TEXT_IDS = dict(vocab_size=49408, max_position_embeddings=77, bos_token_id=49406, eos_token_id=49407, pad_token_id=49407)


@pytest.fixture(scope="module")
def text_towers(ops):  # noqa: F811
    from imagharmony_b200.clip import ClipTextTower
    from oracle import clip_ref as R
    return {"CLIP ViT-L text": _tower(ClipTextTower, _hf_meta("CLIPTextModel", "CLIPTextConfig", **TEXT_IDS, **R.TEXT_L), 5),
            "OpenCLIP bigG text": _tower(ClipTextTower, _hf_meta("CLIPTextModelWithProjection", "CLIPTextConfig",
                                                                 **TEXT_IDS, **R.TEXT_BIGG), 6)}


@pytest.fixture(scope="module")
def vision_tower(ops):  # noqa: F811
    from imagharmony_b200.clip import ClipVisionTower
    from oracle import clip_ref as R
    return _tower(ClipVisionTower, _hf_meta("CLIPVisionModelWithProjection", "CLIPVisionConfig", **R.VISION_BIGG), 7)


def _ids(B, seed):
    """Prompts of several lengths padded with the end-of-text token, and one that fills all 77 positions."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 49406, (B, 77), generator=g)
    ids[:, 0] = 49406
    for b in range(B):
        if b % 4 != 3:
            ids[b, 5 + 13 * b % 70:] = 49407
    return ids


@pytest.mark.parametrize("B", [1, 2, 8])
def test_clip_text_census(ops, text_towers, monkeypatch, B):  # noqa: F811
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    for name, tower in text_towers.items():
        out = tower(_ids(B, B))
        assert out.penultimate.shape == (B, 77, tower.cfg.hidden_size)
    monkeypatch.undo()
    assert {"embed_tokens", "attention_generic"} <= {r["op"] for r in c.rows.values()}
    assert all("causal" in r["shape"] for r in c.rows.values() if r["op"] == "attention_generic")
    _done(c, f"CLIP text towers batch {B}")


@pytest.mark.parametrize("B", [1, 4])
def test_clip_vision_census(ops, vision_tower, monkeypatch, B):  # noqa: F811
    px = torch.randn(B, 3, 224, 224, generator=_gen("vision", B))
    rows = vision_tower.patch_rows(px)
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    out = vision_tower.forward_rows(rows, B, output_hidden_states=True)
    monkeypatch.undo()
    assert out.hidden_states[-2].shape == (B, 257, 1664) and out.image_embeds.shape == (B, 1280)
    assert any(r["op"] == "attention_generic" and "257x257 d104/104" in r["shape"] for r in c.rows.values())
    _done(c, f"CLIP ViT-bigG vision batch {B}")


RESIZE_CASES = [(1024, 1024), (1216, 832), (640, 1536), (160, 200)]


@pytest.mark.parametrize("height,width", RESIZE_CASES, ids=[f"{h}x{w}" for h, w in RESIZE_CASES])
def test_clip_scorer_resize_census(ops, text_towers, vision_tower, monkeypatch, height, width):  # noqa: F811
    from imagharmony_b200.clip import ClipScorer
    scorer = ClipScorer(vision_tower, text_towers["OpenCLIP bigG text"])
    scorer.set_prompt(input_ids=_ids(1, 11))
    imgs = (torch.rand(4, 3, height, width, generator=_gen("score", height, width)) * 2.2 - 1.1).half().cuda()
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    scores = scorer.score_images(imgs)
    monkeypatch.undo()
    assert scores.shape == (4,) and bool(torch.isfinite(scores).all())
    assert any(r["op"] == "resize_patchify" and r["shape"] == f"4x3x{height}x{width}->224" for r in c.rows.values())
    _done(c, f"ClipScorer resize {height}x{width}")


# ---------------------------------------------------------------------------------------------------------------------
# adapter modules and the UNet with the IP-Adapter Plus processors
# ---------------------------------------------------------------------------------------------------------------------
def _random_module(m, seed):
    from imagharmony_b200.weights import random_state_dict, shapes_of
    m.load_state_dict(random_state_dict(shapes_of(m), seed))
    return m.half().cuda().eval()


@pytest.fixture(scope="module")
def adapters(ops):  # noqa: F811
    from imagharmony_b200.adapter import HarmonyAttention, ImageProjModel, Resampler
    from imagharmony_b200.config import HARMONY_DEFAULT as h
    ha = HarmonyAttention(image_hidden_size=h.image_hidden_size, text_context_dim=h.text_context_dim,
                          inter_dim=h.inter_dim, cross_heads=h.cross_heads, reshape_blocks=h.reshape_blocks,
                          cross_value_dim=h.cross_value_dim, scale=h.scale)
    proj = ImageProjModel(cross_attention_dim=2048, clip_embeddings_dim=h.image_hidden_size, clip_extra_context_tokens=4)
    kw = dict(dim=1280, depth=4, dim_head=64, heads=20, num_queries=16, embedding_dim=1664, output_dim=2048, ff_mult=4)
    res = Resampler(**kw)                                                        # IPAdapterPlusXL.init_proj
    # the Resampler's options: position embedding of the 257 tokens and mean-pooled extra latents
    pooled = Resampler(**kw, apply_pos_emb=True, num_latents_mean_pooled=4)
    return _random_module(ha, 8), _random_module(proj, 9), _random_module(res, 10), _random_module(pooled, 11)


@pytest.mark.parametrize("B", [1, 2, 4])
def test_adapter_census(ops, adapters, monkeypatch, B):  # noqa: F811
    from imagharmony_b200.config import HARMONY_DEFAULT as h
    ha, proj, res, pooled = adapters
    g = _gen("adapters", B)
    img = torch.randn(B, h.image_hidden_size, generator=g).half().cuda()
    text = torch.randn(2 * B, 77, h.text_context_dim, generator=g).half().cuda()
    hidden = torch.randn(B, 257, 1664, generator=g).half().cuda()
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    tokens = proj(ha(text, img, add_to=img))
    plus = res(hidden)
    plus_pooled = pooled(hidden)
    monkeypatch.undo()
    assert tokens.shape == (B, 4, 2048) and plus.shape == (B, 16, 2048) and plus_pooled.shape == (B, 20, 2048)
    labels = {(r["op"], r["shape"]) for r in c.rows.values()}
    assert ("attention", f"B{B} H20 16x273 n_ip=0") in labels, "the Resampler's 16-query attention over 257 + 16 keys"
    assert {"attention_small", "add_bcast", "mean_tokens"} <= {op for op, _ in labels}
    _done(c, f"adapters batch {B}")


@pytest.fixture(scope="module")
def sdxl_unet_plus(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.ip_adapter import IPAdapterPlusXL
    cfg = dataclasses.replace(SDXL_BASE, num_ip_tokens=16)
    with torch.device("meta"):
        shapes = shapes_of(UNet2DConditionModel(cfg))
    unet = UNet2DConditionModel.from_state_dict(cfg, random_state_dict(shapes, 12, device="cuda"), device="cuda")
    # the processors IPAdapterPlusXL installs; set_ip_adapter zeroes them (load_ip_adapter fills them), so random
    # to_k_ip / to_v_ip stand in for the checkpoint: with zeros the image branch would add nothing a bar can see
    IPAdapterPlusXL.set_ip_adapter(types.SimpleNamespace(pipe=types.SimpleNamespace(unet=unet), num_tokens=16,
                                                         device="cuda"))
    procs = torch.nn.ModuleList(unet.attn_processors.values())
    procs.load_state_dict(random_state_dict(shapes_of(procs), 13, device="cuda"))
    unet.finalize()
    return unet


PLUS_CASES = [(1024, 1024), (832, 1216)]


@pytest.mark.parametrize("height,width", PLUS_CASES, ids=[f"{h}x{w}" for h, w in PLUS_CASES])
def test_ip_adapter_plus_unet_census(ops, sdxl_unet_plus, monkeypatch, height, width):  # noqa: F811
    unet = sdxl_unet_plus
    B = 2
    g = _gen("plus", height, width)
    sample = torch.randn(B, 4, height // 8, width // 8, generator=g).half().cuda()
    ehs, te, tid = _conditioning(unet.config, B, height, width, g)
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    with torch.no_grad():
        out = unet(sample, torch.full((B,), 501.0, device="cuda"), ehs, te, tid)
    monkeypatch.undo()
    assert out.shape == (B, 4, height // 8, width // 8)
    assert any(r["op"] == "attention" and "n_ip=16" in r["shape"] for r in c.rows.values()), \
        "the IP-Adapter Plus layers must run their decoupled attention over 77 + 16 keys"
    _done(c, f"UNet with IP-Adapter Plus processors {height}x{width}")
