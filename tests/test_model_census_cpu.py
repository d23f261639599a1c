"""The census plumbing of test_model_census_gpu.py without a GPU: every public op is classified (a census reference, a
host helper, or a scheduler step kernel with its own bit-exact test); each model the product runs besides the UNet and
the untiled VAE decoder runs on its TINY configuration at a non-square size under the recorder, with the stand-in ops
of tests/fake_ops*.py, every op it calls has a reference that reads every argument of the op and none is beyond its
bar (a reference blind to `relu` fails both ways); the new comparators reject an output one element of which is 2 fp16
ulps off (1 ulp for the bit-exact ones), and the ReLU-aware ones an output without the ReLU or with it before the
residual."""
import inspect
import math
import os

import pytest
import torch

import census
import fake_ops
import fake_ops_controlnet
import fake_ops_img2img
import fake_ops_inpaint9
import fake_ops_multi_controlnet
from img2img_ref import posterior_noise_ref
from test_unet_census_cpu import _nudge, _rnd
from test_wiring_cpu import _build, patched  # noqa: F401  (fixture)

HERE = os.path.dirname(os.path.abspath(__file__))


# ---------------------------------------------------------------------------------------------------------------------
# classification
# ---------------------------------------------------------------------------------------------------------------------
def test_every_op_is_classified_once():
    from imagharmony_b200 import ops
    names = set(census.op_names(ops))
    groups = {"REFERENCES": set(census.REFERENCES), "EXEMPT": census.EXEMPT, "STEP_KERNELS": set(census.STEP_KERNELS)}
    for n in sorted(names):
        homes = [g for g, members in groups.items() if n in members]
        assert len(homes) == 1, f"ops.{n} is in {homes or 'none'} of REFERENCES / EXEMPT / STEP_KERNELS"
    for g, members in groups.items():
        assert members <= names, f"{g} lists ops that do not exist: {sorted(members - names)}"


def test_every_step_kernel_names_an_existing_test():
    for op, where in census.STEP_KERNELS.items():
        path, name = where.split("::")
        with open(os.path.join(HERE, path)) as f:
            assert f"\ndef {name}(" in f.read(), f"{op}: {where} does not exist"


# ---------------------------------------------------------------------------------------------------------------------
# plumbing: each model under the recorder on the stand-in ops
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def stand_ins(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as real_ops
    for mod in (fake_ops_img2img, fake_ops_inpaint9, fake_ops_multi_controlnet):
        for name in mod.NAMES:
            monkeypatch.setattr(real_ops, name, getattr(mod, name))
    # not fake_ops_controlnet.conv3x3: it hides conv3x3's keyword arguments, and the forwards here pass no `out`
    for name in ("conv3x3_small", "controlnet_add_residuals"):
        monkeypatch.setattr(real_ops, name, getattr(fake_ops_controlnet, name))
    yield


def _vae_tiled_decode():
    from imagharmony_b200.config import TINY_VAE
    from test_vae_cpu import _pair
    native, _ = _pair(TINY_VAE, seed=4)
    native.use_tiling = True
    z = torch.randn(1, 4, 14, 11, generator=torch.Generator().manual_seed(2)) * TINY_VAE.scaling_factor * 3
    return lambda: native.decode(z), {"im2col3x3_nchw", "linear", "conv3x3", "groupnorm", "softmax_rows_masked_"}


def _vae_tiled_encode():
    from imagharmony_b200.config import TINY_VAE
    from test_img2img_cpu import _encoder_pair, _image
    native, _ = _encoder_pair(TINY_VAE, seed=4)
    native.use_tiling = True
    x = _image(1, 3, 104, 88, seed=2)                        # tiles at 0 / 48 / 96 rows, 0 / 48 columns

    def run():
        from imagharmony_b200 import ops
        m = native.encode_moments_nhwc(x)
        g = torch.Generator().manual_seed(5)
        eps = torch.randn(1, 4, m.shape[1], m.shape[2], generator=g)
        for n in (1, 4):
            noise = torch.randn(n, 4, m.shape[1], m.shape[2], generator=g).half()
            ops.vae_posterior_noise(m, eps, noise, 4, TINY_VAE.scaling_factor, 3.0)
    return run, {"conv3x3_down", "vae_posterior_noise", "conv3x3", "groupnorm"}


def _controlnet(k):
    def build():
        from imagharmony_b200.config import TINY, TINY_CONTROLNET
        from test_controlnet_cpu import _cn_pair
        unet, _ = _build(TINY, 0)
        net, _ = _cn_pair(TINY_CONTROLNET, 0)
        g = torch.Generator().manual_seed(3)
        n, h, w = 2, 16, 24
        sample = torch.randn(2 * n, 4, h, w, generator=g)
        ehs = torch.randn(2 * n, 77 + TINY.num_ip_tokens, TINY.cross_attention_dim, generator=g)
        te = torch.randn(2 * n, TINY.pooled_embed_dim, generator=g)
        tid = torch.tensor([[h * 8., w * 8., 0., 0., h * 8., w * 8.]] * 2 * n)
        t = torch.full((2 * n,), 321.0)

        def run():
            for guess in (False, True):
                rows = slice(n, 2 * n) if guess else slice(0, 2 * n)          # guess mode: the conditional half only
                outs = []
                for j in range(k):
                    img = torch.rand(rows.stop - rows.start, 3, 8 * h, 8 * w, generator=g)
                    outs.append(net(sample[rows], t[rows], ehs[rows, :77].contiguous(), controlnet_cond=img,
                                    conditioning_scale=0.7 - 0.2 * j, guess_mode=guess, text_embeds=te[rows],
                                    time_ids=tid[rows]))
                unet(sample, t, ehs, te, tid, controlnet_residuals=(outs[0] if k == 1 else outs, n if guess else 0))
        want = {"conv3x3_small", "controlnet_add_residuals" if k == 1 else "controlnet_add_residuals_multi"}
        return run, want
    return build


def _unet9():
    import dataclasses
    from imagharmony_b200.config import TINY
    native, _ = _build(dataclasses.replace(TINY, in_channels=9), 0)
    g = torch.Generator().manual_seed(1)
    B, h, w = 2, 16, 24
    sample, cond = torch.randn(B, 4, h, w, generator=g), torch.randn(B, 5, h, w, generator=g)
    ehs = torch.randn(B, 77 + TINY.num_ip_tokens, TINY.cross_attention_dim, generator=g)
    te = torch.randn(B, TINY.pooled_embed_dim, generator=g)
    tid = torch.tensor([[h * 8., w * 8., 0., 0., h * 8., w * 8.]] * B)
    return lambda: native(sample, torch.full((B,), 321.0), ehs, te, tid, cond=cond), {"im2col3x3_nchw_cat"}


def _clip_text():
    pytest.importorskip("transformers")
    from imagharmony_b200.clip import ClipTextTower
    from oracle.clip_ref import hf_text_model
    towers = [ClipTextTower.from_hf(hf_text_model(3, proj, vocab_size=100, eos_token_id=99, hidden_size=64,
                                                  intermediate_size=160, num_hidden_layers=2, num_attention_heads=4,
                                                  hidden_act=act, projection_dim=48), device="cpu")
              for proj, act in ((False, "quick_gelu"), (True, "gelu"))]
    ids = torch.randint(0, 98, (3, 77), generator=torch.Generator().manual_seed(5))
    ids[0, 9:] = 99                                        # padded with the end-of-text token

    def run():
        for t in towers:
            t(ids)
    return run, {"embed_tokens", "attention_generic", "layernorm", "linear", "linear_small"}


def _clip_vision():
    pytest.importorskip("transformers")
    from imagharmony_b200.clip import ClipScorer, ClipTextTower, ClipVisionTower
    from oracle.clip_ref import hf_text_model, hf_vision_model
    vision = ClipVisionTower.from_hf(hf_vision_model(4, hidden_size=208, intermediate_size=320, num_hidden_layers=2,
                                                     num_attention_heads=2, hidden_act="gelu", projection_dim=40,
                                                     image_size=56, patch_size=14), device="cpu")
    text = ClipTextTower.from_hf(hf_text_model(3, True, vocab_size=100, eos_token_id=99, hidden_size=64,
                                               intermediate_size=160, num_hidden_layers=2, num_attention_heads=4,
                                               hidden_act="gelu", projection_dim=40), device="cpu")
    scorer = ClipScorer(vision, text)
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(0, 98, (1, 77), generator=g)
    ids[0, 12:] = 99

    def run():
        scorer.set_prompt(input_ids=ids)
        for shape in ((3, 3, 152, 104), (1, 3, 40, 48)):                 # a downscaling and an upscaling area average
            scorer.score_images((torch.rand(shape, generator=g) * 2.2 - 1.1).half())
    return run, {"resize_patchify", "attention_generic", "embed_tokens"}


def _adapters():
    from imagharmony_b200.adapter import HarmonyAttention, ImageProjModel, Resampler
    from imagharmony_b200.config import HARMONY_TINY as h
    torch.manual_seed(0)
    ha = HarmonyAttention(image_hidden_size=h.image_hidden_size, text_context_dim=h.text_context_dim,
                          inter_dim=h.inter_dim, cross_heads=h.cross_heads, reshape_blocks=h.reshape_blocks,
                          cross_value_dim=h.cross_value_dim).half()
    proj = ImageProjModel(128, h.image_hidden_size, 4).half()
    res = Resampler(dim=128, depth=2, dim_head=64, heads=2, num_queries=16, embedding_dim=80, output_dim=96, ff_mult=2,
                    apply_pos_emb=True, num_latents_mean_pooled=2).half()
    g = torch.Generator().manual_seed(7)

    def run():
        for B in (1, 3):
            img = torch.randn(B, h.image_hidden_size, generator=g).half()
            text = torch.randn(2 * B, 77, h.text_context_dim, generator=g).half()
            proj(ha(text, img, add_to=img))
            res(torch.randn(B, 41, 80, generator=g).half())
    return run, {"attention_small", "add_bcast", "mean_tokens", "attention", "linear_small", "layernorm"}


def _taesd():
    from test_taesd_cpu import SMALL, _cfg, _pair
    native, _ = _pair(_cfg(**SMALL), seed=3)
    z = torch.randn(1, 4, 6, 9, generator=torch.Generator().manual_seed(8)) * 4
    return lambda: native.decode(z), {"im2col3x3_nchw", "linear", "conv3x3", "upsample2x", "nhwc_to_nchw"}


MODELS = {"vae-tiled-decode": _vae_tiled_decode, "vae-tiled-encode": _vae_tiled_encode,
          "controlnet": _controlnet(1), "multi-controlnet": _controlnet(2), "unet9": _unet9,
          "clip-text": _clip_text, "clip-vision": _clip_vision, "adapters": _adapters, "taesd": _taesd}


def _run_model(model, monkeypatch, references=census.REFERENCES):
    from imagharmony_b200 import ops
    run, want = MODELS[model]()
    c = census.Census(ops, references=references).install(monkeypatch)
    with torch.no_grad():
        run()
    return c, want


@pytest.mark.parametrize("model", list(MODELS))
def test_every_op_of_the_model_has_a_reference(stand_ins, monkeypatch, model):
    c, want = _run_model(model, monkeypatch)
    print(c.report(model))
    called = {r["op"] for r in c.rows.values()}
    assert want <= called, f"{model}: {sorted(want - called)} ran unchecked"
    assert called <= set(census.REFERENCES)
    assert not c.unread(), f"{model}: arguments no reference reads: {c.unread()}"
    assert not c.failures(), c.report(model)
    assert all(r["checked"] == r["calls"] for r in c.rows.values())
    if model == "taesd":              # the ReLU epilogue on the GEMM (conv_in) and on the convs, and the scaled conv_out
        shapes = {(r["op"], f) for r in c.rows.values() for f in r["shape"].split()}
        assert {("linear", "relu"), ("conv3x3", "relu"), ("conv3x3", "alpha=2")} <= shapes


def test_a_reference_that_ignores_an_argument_fails_the_census(stand_ins, monkeypatch):
    """ref_linear handed a copy of its arguments with `relu` forced off: the guard names linear(relu), and the ReLU
    rows of the tiny decoder are beyond their bar."""
    def blind(res, p):
        return census.ref_linear(res, {**{k: p[k] for k in p if k != "relu"}, "relu": False})
    c, _ = _run_model("taesd", monkeypatch, references=dict(census.REFERENCES, linear=blind))
    assert c.unread() == ["linear(relu)"]
    assert [r["op"] for r in c.failures()] == ["linear"]


# ---------------------------------------------------------------------------------------------------------------------
# comparator sensitivity
# ---------------------------------------------------------------------------------------------------------------------
def _rejects(ref, good, p, ulps=2):
    assert ref(good, p) <= 1.0
    assert ref(_nudge(good, ulps), p) > 1.0


def test_new_comparators_reject_two_ulps():
    # conv3x3_down at a VAE encoder width; alpha as in its scaled stream
    x, w, b = _rnd(1, 16, 24, 128, seed=1), _rnd(128, 9 * 128, scale=(9 * 128) ** -0.5, seed=2), _rnd(128, seed=3)
    for alpha in (1.0, 2.0 ** -7):
        p = dict(x=x, w_packed=w, bias=b, out=None, tile_n=0, alpha=alpha)
        _rejects(census.ref_conv3x3_down, fake_ops_img2img.conv3x3_down(x, w, b, alpha=alpha), p)

    # conv3x3_small: the NCHW control image (3 -> 16, SiLU) and an NHWC stride-2 layer
    img = torch.rand(1, 3, 40, 56, generator=torch.Generator().manual_seed(4)).half()
    for xs, cin, cout, stride, nchw in ((img, 3, 16, 1, True), (_rnd(1, 20, 28, 32, seed=5), 32, 96, 2, False)):
        ws, bs = _rnd(cout, 9 * cin, scale=(9 * cin) ** -0.5, seed=6), _rnd(cout, scale=0.5, seed=7)
        p = dict(x=xs, w_packed=ws, bias=bs, stride=stride, silu=True, nchw=nchw, out=None)
        _rejects(census.ref_conv3x3_small, fake_ops_controlnet.conv3x3_small(xs, ws, bs, stride=stride, silu=True,
                                                                              nchw=nchw), p)

    # attention_generic: a CLIP text layer (causal, head_dim 64) and a ViT-bigG one (head_dim 104); with V >= 0,
    # P @ |V| is the output and the bar stays below 1 ulp
    for B, H, N, d, causal in ((2, 2, 77, 64, True), (1, 2, 257, 104, False)):
        q, k = _rnd(B * N, H * d, scale=1.5, seed=8), _rnd(B * N, H * d, scale=1.5, seed=9)
        v = _rnd(B * N, H * d, seed=10).abs()
        p = dict(q=q, k=k, v=v, B=B, H=H, Nq=N, Nk=N, dqk=d, dv=d, scale=d ** -0.5, causal=causal, out=None)
        _rejects(census.ref_attention_generic, fake_ops.attention_generic(q, k, v, B, H, N, N, d, d, d ** -0.5, causal), p)

    # attention_small at HarmonyAttention's shape (10 heads, 8 queries, 77 keys, head_dim 32, value dim 64).  V close to
    # one constant: P @ |V - out| is small, so the score term cannot hide the nudge; the fp16 store of p costs 2^-11
    # P @ |V| = 0.75 ulp of outputs near 1.5
    B, H, Nq, Nk, dqk, dv = 2, 10, 8, 77, 32, 64
    q, k = _rnd(B * Nq, H * dqk, scale=0.5, seed=11), _rnd(B * Nk, H * dqk, scale=0.5, seed=12)
    v = (1.5 + 0.01 * _rnd(B * Nk, H * dv, seed=13).float()).half()
    p = dict(q=q, k=k, v=v, B=B, H=H, Nq=Nq, Nk=Nk, dqk=dqk, dv=dv, scale=math.sqrt(dqk), out=None)
    _rejects(census.ref_attention_small, fake_ops.attention_small(q, k, v, B, H, Nq, Nk, dqk, dv, math.sqrt(dqk)), p)

    # mean_tokens over the 257 CLIP tokens
    xm = _rnd(2, 257, 1280, seed=14)
    _rejects(census.ref_mean_tokens, xm.float().mean(dim=1).half(), dict(x=xm, out=None))

    # resize_patchify of 1216 x 832 candidates (half size here) to 224^2
    from imagharmony_b200.clip import CLIP_MEAN, CLIP_STD
    imr = (torch.rand(2, 3, 608, 416, generator=torch.Generator().manual_seed(15)) * 2.2 - 1.1).half()
    p = dict(img=imr, size=224, patch=14, kpad=592, mean=CLIP_MEAN, std=CLIP_STD, out=None)
    _rejects(census.ref_resize_patchify, fake_ops.resize_patchify(imr, 224, 14, 592, CLIP_MEAN, CLIP_STD), p)

    # vae_posterior_noise: one image's moments for 4 noise draws, fp32 eps
    g = torch.Generator().manual_seed(16)
    mom = (torch.randn(1, 13, 11, 16, generator=g) * 2).half()
    eps, noise = torch.randn(1, 4, 13, 11, generator=g), torch.randn(4, 4, 13, 11, generator=g).half()
    p = dict(moments=mom, eps=eps, noise=noise, channels=4, scaling_factor=0.13025, sigma=3.0742, out=None)
    _rejects(census.ref_vae_posterior_noise, posterior_noise_ref(mom, eps, noise, 4, 0.13025, 3.0742).contiguous(), p)


def _bound(fn, *a, **k):
    b = inspect.signature(fn).bind(*a, **k)
    b.apply_defaults()
    return dict(b.arguments)


def test_relu_comparators_reject_a_missing_or_misplaced_relu():
    """ref_linear / ref_conv3x3 with relu=True (IH_EPI_RELU: relu(alpha * acc + bias + residual)) reject the output
    without the ReLU, the output with the ReLU before the residual, and one element 2 fp16 ulps off."""
    g = torch.Generator().manual_seed(20)
    # linear: conv_in's GEMM form (im2col rows of 64) with a residual and alpha
    x, w, b, r = _rnd(96, 64, seed=21), _rnd(64, 64, scale=0.125, seed=22), _rnd(64, scale=0.5, seed=23), _rnd(96, 64, seed=24)
    cases = [(census.ref_linear, fake_ops.linear, (x, w, b), dict(residual=r, alpha=0.5))]
    # conv3x3: a TinyBlock's third conv (residual) and a stride-2 conv with a residual and alpha
    for B, H, W, C, stride, alpha in ((2, 6, 10, 64, 1, 1.0), (1, 8, 12, 128, 2, 2.0)):
        xc = (torch.randn(B, H, W, C, generator=g)).half()
        wc = (torch.randn(C, 9 * C, generator=g) * (9 * C) ** -0.5).half()
        bc, rc = (torch.randn(C, generator=g) * 0.5).half(), torch.randn(B, H // stride, W // stride, C, generator=g).half()
        cases.append((census.ref_conv3x3, fake_ops.conv3x3, (xc, wc, bc), dict(residual=rc, stride=stride, alpha=alpha)))
    for ref, fn, args, kw in cases:
        p = _bound(fn, *args, **kw, relu=True)
        good = fn(*args, **kw, relu=True)
        assert ref(good, p) <= 1.0
        assert ref(fn(*args, **kw), p) > 1.0, "no ReLU"
        pre = fn(*(a.float() for a in args), **dict(kw, residual=None))              # fp32: alpha * acc + bias
        assert ref((torch.relu(pre) + kw["residual"].float()).half(), p) > 1.0, "ReLU before the residual"
        assert ref(_nudge(good, 2), p) > 1.0, "2 ulps"


def test_bit_exact_comparators_reject_one_ulp():
    tok, pos = _rnd(1000, 768, seed=1), _rnd(77, 768, seed=2)
    ids = torch.randint(-3, 1003, (2, 77), generator=torch.Generator().manual_seed(3), dtype=torch.int32)  # clamped
    p = dict(ids=ids, tok_emb=tok, pos_emb=pos, out=None)
    good = (tok[ids.long().clamp(0, 999)].float() + pos.float()[None]).half().reshape(2 * 77, 768)
    _rejects(census.ref_embed_tokens, good, p, ulps=1)

    a, b = _rnd(2, 257, 1664, seed=4), _rnd(257, 1664, seed=5)
    _rejects(census.ref_add_bcast, (a.float() + b.float()[None]).half(), dict(a=a, b=b, out=None), ulps=1)

    x0, x1 = _rnd(2, 4, 19, 13, seed=6), _rnd(2, 5, 19, 13, seed=7)
    _rejects(census.REFERENCES["im2col3x3_nchw_cat"], fake_ops_inpaint9.im2col3x3_nchw_cat(x0, x1, 128),
             dict(x0=x0, x1=x1, kpad=128, out=None), ulps=1)

    # guess-mode injection: residuals for the last 2 of 4 images, added from row 2 * (rows per image) on
    skips = [_rnd(4, 10, 12, 64, seed=8), _rnd(4, 5, 6, 128, seed=9)]
    res = [[_rnd(2, 10, 12, 64, seed=10 + j), _rnd(2, 5, 6, 128, seed=12 + j)] for j in range(2)]
    scales = [torch.tensor([0.7, 0.4]), torch.tensor([0.3, 1.0])]
    row0s = [2 * 120, 2 * 30]
    single = [s.clone() for s in skips]
    fake_ops_controlnet.controlnet_add_residuals(single, res[0], scales[0], row0s)
    multi = [s.clone() for s in skips]
    fake_ops_multi_controlnet.controlnet_add_residuals_multi(multi, res, scales, row0s)
    for ref, got, p in ((census.ref_controlnet_add_residuals, single,
                         dict(skips=skips, residuals=res[0], scale=scales[0], skip_row0s=row0s)),
                        (census.ref_controlnet_add_residuals_multi, multi,
                         dict(skips=skips, residuals_per_net=res, scales_per_net=scales, skip_row0s=row0s))):
        assert ref(got, p) == 0.0
        for i in range(2):
            bad = list(got)
            bad[i] = _nudge(got[i], 1)
            assert ref(bad, p) == float("inf")
        outside = list(got)                                   # a write outside the injected rows
        outside[0] = got[0].clone()
        outside[0].view(-1, 64)[0, 0] = -outside[0].view(-1, 64)[0, 0] - 1
        assert ref(outside, p) == float("inf")
