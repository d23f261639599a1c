"""GPU tests of the tiny autoencoder decoder (imagharmony_b200.taesd) and the ReLU epilogue it runs on (IH_EPI_RELU):
the epilogue against torch fp32 within fp16-ulp bounds at every 64-channel resolution the decoder sees, IH_EPI_NONE
through the widened ih_conv2d_scaled_f16 bit-equal to the plain conv, the decoder against the fp32 oracle
(tests/taesd_ref.py) at every SDXL bucket and with a NaN latent, a launch census of one decode, the PNS judge with the tiny decode and one
IPAdapterXL.generate to PIL images."""
import pytest
import torch
import torch.nn.functional as F

from fp16_ulps import close_ulps

pytestmark = pytest.mark.gpu

# SDXL resolution buckets (height, width); the tiny decoder runs 64-channel convs at 1/8, 1/4, 1/2 and full size
BUCKETS = [(1024, 1024), (1152, 896), (1216, 832), (1344, 768), (1536, 640),
           (896, 1152), (832, 1216), (768, 1344), (640, 1536)]
EPS32 = 2.0 ** -24


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _rnd(*shape, scale=1.0, seed=0):
    return (torch.randn(*shape, generator=torch.Generator("cpu").manual_seed(seed)) * scale).half().cuda()


def _conv_ref(x, w, bias, residual, alpha):
    """fp32 relu(alpha * conv(x) + bias + residual) and the accumulation allowance: K 2^-24 alpha (|x| * |w|), K = 9 Cin
    roundings of a running fp32 sum in the kernel and in cuDNN each (fp32 epilogue: 4 more roundings of |out|)."""
    xn = x.float().permute(0, 3, 1, 2)
    y = F.conv2d(xn, w.float(), None, padding=1).permute(0, 2, 3, 1) * alpha
    mag = F.conv2d(xn.abs(), w.float().abs(), None, padding=1).permute(0, 2, 3, 1) * abs(alpha)
    if bias is not None:
        y = y + bias.float()
    if residual is not None:
        y = y + residual.float()
    K = 9 * x.shape[-1]
    return torch.relu(y), (2 * K * EPS32 * mag + 4 * EPS32 * y.abs()).double()


@pytest.mark.parametrize("H,W", BUCKETS[:5])
def test_relu_conv_epilogue_at_decoder_resolutions(H, W):
    """Cin = Cout = 64 at each resolution the decoder sees for this bucket and its transpose, with and without bias,
    with a residual and with alpha != 1; batch 8 at the two smaller sizes."""
    from imagharmony_b200 import ops
    C = 64
    w = _rnd(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
    wp = ops.pack_conv3x3_weight(w)
    b = _rnd(C, scale=0.5, seed=2)
    for hh, ww in ((H, W), (W, H)):
        for k, f in enumerate((8, 4, 2, 1)):
            for B in ((1, 8) if f >= 4 else (1,)):
                x = _rnd(B, hh // f, ww // f, C, seed=3 + k)
                r = _rnd(B, hh // f, ww // f, C, seed=4 + k)
                for bias, res, alpha in ((b, None, 1.0), (None, None, 1.0), (b, r, 1.0), (None, r, 0.5), (b, r, 2.0)):
                    out = ops.conv3x3(x, wp, bias, residual=res, alpha=alpha, relu=True)
                    want, slack = _conv_ref(x, w, bias, res, alpha)
                    assert (out >= 0).all()
                    close_ulps(out, want, f"relu conv {B}x{hh // f}x{ww // f} bias={bias is not None} "
                               f"res={res is not None} alpha={alpha}", ulps=0.5, slack=slack)
                    del out, want, slack
    torch.cuda.synchronize()


def test_relu_gemm_epilogue_conv_in_form():
    """conv_in as the decoder runs it: 4 latent channels -> im2col rows of 64 -> GEMM with IH_EPI_RELU (alpha, bias,
    residual); the flag through ih_gemm_scaled_f16 with other flags is refused."""
    from imagharmony_b200 import _lib, ops
    from imagharmony_b200._lib import IHError
    w = _rnd(64, 4, 3, 3, scale=36 ** -0.5, seed=5)
    wg = torch.zeros(64, 64, dtype=torch.float16, device="cuda")
    wg[:, :36] = w.reshape(64, 36)
    b = _rnd(64, scale=0.5, seed=6)
    for B, h, wd in ((1, 128, 128), (8, 80, 192), (3, 7, 9)):
        z = _rnd(B, 4, h, wd, scale=2.0, seed=B)
        a = ops.im2col3x3_nchw(z, 64)
        res = _rnd(B * h * wd, 64, seed=7)
        for bias, r, alpha in ((b, None, 1.0), (None, None, 1.0), (b, res, 0.5)):
            out = ops.linear(a, wg, bias, residual=r, alpha=alpha, relu=True)
            y = (a.float() @ wg.float().t()) * alpha
            mag = (a.float().abs() @ wg.float().abs().t()) * alpha
            y = y + (bias.float() if bias is not None else 0) + (r.float() if r is not None else 0)
            close_ulps(out, torch.relu(y), f"relu gemm {B}x{h}x{wd}", ulps=0.5,
                       slack=(2 * 64 * EPS32 * mag + 4 * EPS32 * y.abs()).double())
    a = ops.im2col3x3_nchw(_rnd(1, 4, 8, 8, seed=9), 64)
    out = torch.empty(64, 64, dtype=torch.float16, device="cuda")
    lib = _lib.load()
    rc = lib.ih_gemm_scaled_f16(a.data_ptr(), 64, wg.data_ptr(), None, None, 0, out.data_ptr(), 64, 64, 64, 64,
                                ops.EPI_RELU | ops.EPI_SILU, 1.0, ops._stream())
    assert rc < 0 and b"IH_EPI_RELU" in lib.ih_last_error()
    with pytest.raises(IHError):
        ops.linear(a, wg, relu=True, silu=True)


def test_conv_scaled_epi_none_is_bit_equal_to_the_plain_conv():
    """ih_conv2d_scaled_f16 with its new trailing argument IH_EPI_NONE computes what it did: bit-equal to ops.conv3x3
    (ih_conv2d_f16 at alpha 1; the same entry point at alpha 0.125), stride 1 and 2, with a residual; an unknown
    epilogue is refused."""
    from imagharmony_b200 import _lib, ops
    lib = _lib.load()
    for B, H, W, Cin, Cout, stride in ((2, 40, 24, 64, 64, 1), (1, 128, 128, 128, 256, 1), (2, 32, 48, 64, 128, 2)):
        x = _rnd(B, H, W, Cin, seed=H)
        wp = ops.pack_conv3x3_weight(_rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=W))
        b = _rnd(Cout, seed=Cin)
        r = _rnd(B, H // stride, W // stride, Cout, seed=Cout)
        for alpha in (1.0, 0.125):
            want = ops.conv3x3(x, wp, b, residual=r, stride=stride, alpha=alpha)
            got = torch.empty_like(want)
            rc = lib.ih_conv2d_scaled_f16(x.data_ptr(), wp.data_ptr(), b.data_ptr(), r.data_ptr(), got.data_ptr(), B, H,
                                          W, Cin, Cout, stride, alpha, ops._stream(), ops.EPI_NONE)
            _lib.check(rc, "ih_conv2d_scaled_f16")
            assert torch.equal(got, want), (B, H, W, Cin, Cout, stride, alpha)
    rc = lib.ih_conv2d_scaled_f16(x.data_ptr(), wp.data_ptr(), None, None, got.data_ptr(), B, H, W, Cin, Cout, stride,
                                  1.0, ops._stream(), ops.EPI_SILU)
    assert rc < 0
    torch.cuda.synchronize()


def _models(cfg, seed):
    from imagharmony_b200.taesd import AutoencoderTinyDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from taesd_ref import AutoencoderTinyRef
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderTinyRef(cfg))
    sd = random_state_dict(shapes, seed)
    native = AutoencoderTinyDecoder.from_state_dict(cfg, sd, device="cuda")
    ref32 = AutoencoderTinyRef(cfg)
    ref32.load_state_dict({k: v.float() for k, v in sd.items()})
    eager16 = AutoencoderTinyRef(cfg)
    eager16.load_state_dict({k: v.float() for k, v in sd.items()})
    return native, ref32.cuda().eval(), eager16.half().cuda().eval()


_MODELS = {}


def _taesdxl():
    from imagharmony_b200.config import TAESDXL
    if "xl" not in _MODELS:
        _MODELS["xl"] = _models(TAESDXL, 11)
    return _MODELS["xl"]


def _check(models, z, what):
    """The bar of test_vae_gpu.py: the native fp16 decoder no further from the fp32 oracle (on the GPU, TF32 off) than
    2x the same oracle evaluated in torch fp16, or 2e-3 of the output's magnitude."""
    native, ref32, eager16 = models
    with torch.no_grad():
        r = ref32.decode(z.float())
        e = eager16.decode(z)
        o = native.decode(z)
    torch.cuda.synchronize()
    e_nat, e_eag, mx = (o.float() - r).abs().max().item(), (e.float() - r).abs().max().item(), r.abs().max().item()
    print(f"[taesd {what}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  max|ref| {mx:.3e}")
    B, _, h, w = z.shape
    assert o.shape == (B, 3, 8 * h, 8 * w) and o.dtype == torch.float16 and torch.isfinite(o).all()
    assert e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
    return o


def test_decoder_small_matches_oracle():
    from imagharmony_b200.config import TAESDXL
    import dataclasses
    small = _models(dataclasses.replace(TAESDXL, num_decoder_blocks=(1, 2, 1, 1)), 12)
    _check(small, _rnd(2, 4, 9, 13, scale=3.0, seed=1), "small 2x9x13")
    _check(_taesdxl(), _rnd(1, 4, 32, 32, scale=3.0, seed=2), "TAESD-XL 256^2")


@pytest.mark.parametrize("H,W", BUCKETS)
def test_decoder_matches_oracle_at_sdxl_buckets(H, W):
    for B in (1, 8):
        _check(_taesdxl(), _rnd(B, 4, H // 8, W // 8, scale=3.0, seed=B), f"B{B} {H}x{W}")
        torch.cuda.empty_cache()


def test_nan_latent_gives_the_nan_footprint_of_the_oracle():
    """One NaN in a latent: the native decode's NaN elements are exactly those of the fp32 oracle (ReLU keeps NaN as
    torch.relu does), the other image of the batch stays NaN-free and everything else is finite."""
    import copy
    native, ref32, _ = _taesdxl()
    z = _rnd(2, 4, 48, 64, scale=3.0, seed=6)
    z[0, 2, 40, 7] = float("nan")          # footprint: 209 x 209 px at image 0's bottom-left
    o = native.decode(z)
    with torch.no_grad():       # on the host: every conv output there reads exactly its 3x3 window
        r = copy.deepcopy(ref32).cpu().decode(z.float().cpu())
    nan_o, nan_r = torch.isnan(o).cpu(), torch.isnan(r)
    print(f"[taesd nan] oracle NaN elements {int(nan_r.sum())}, native {int(nan_o.sum())}")
    assert 0 < nan_r[0].float().mean() < 0.5 and not nan_r[1].any()
    assert torch.equal(nan_o, nan_r)
    assert torch.isfinite(o.cpu()[~nan_r]).all()


def test_decode_launch_census():
    """One decode launches exactly: conv_in (im2col + GEMM), 3 convs per block, per upsample the upsample and its conv,
    conv_out and the NCHW gather.  The tanh clamp is torch elementwise glue and launches nothing of the library."""
    from imagharmony_b200 import ops
    from imagharmony_b200.config import TAESDXL as cfg
    native = _taesdxl()[0]
    z = _rnd(2, 4, 16, 24, seed=3)
    native.decode(z)
    torch.cuda.synchronize()
    ops.launch_count_reset()
    native.decode(z)
    torch.cuda.synchronize()
    n = len(cfg.num_decoder_blocks)
    convs = 1 + 3 * sum(cfg.num_decoder_blocks) + (n - 1) + 1
    assert convs == 35
    assert ops.launch_count() == convs + (n - 1) + 2 == 40


def test_clip_judge_with_tiny_decode():
    """ClipScorer(vision, text, decode=tiny.decode), the cheap PNS judge, against the same towers scoring the fp32
    oracle's decode of the same latents."""
    from imagharmony_b200.clip import ClipScorer, ClipTextTower, ClipVisionTower
    from oracle import clip_ref as R
    native, ref32, _ = _taesdxl()
    hv = R.hf_vision_model(6, hidden_size=256, intermediate_size=512, num_hidden_layers=4, num_attention_heads=4,
                           hidden_act="gelu", projection_dim=64, image_size=224, patch_size=14)
    ht = R.hf_text_model(7, True, hidden_size=128, intermediate_size=256, num_hidden_layers=3, num_attention_heads=2,
                         hidden_act="gelu", projection_dim=64)
    vision, text = ClipVisionTower.from_hf(hv, device="cuda"), ClipTextTower.from_hf(ht, device="cuda")
    ids = torch.full((1, 77), 49407, dtype=torch.int64)
    ids[0, 0] = 49406
    ids[0, 1:9] = torch.tensor([320, 1125, 539, 5567, 15, 2533, 3027, 267])
    tiny = ClipScorer(vision, text, decode=native.decode)
    oracle = ClipScorer(vision, text, decode=lambda lat: ref32.decode(lat.float()).half())
    tiny.set_prompt(input_ids=ids)
    oracle.set_prompt(input_ids=ids)
    lat = _rnd(4, 4, 64, 64, scale=3.0, seed=4)
    got, want = tiny(lat), oracle(lat)
    torch.cuda.synchronize()
    print(f"[taesd judge] tiny {got.tolist()} vs oracle {want.tolist()}")
    assert got.shape == (4,) and torch.allclose(got, want, atol=5e-4)


def test_ip_adapter_generate_pil_with_tiny_vae():
    from PIL import Image
    from imagharmony_b200.config import TINY
    from imagharmony_b200.vae import postprocess
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=2)
    pipe.vae = _taesdxl()[0]
    ip = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4, inference=True)
    ip.image_proj_model.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(ip.image_proj_model), 3).items()})
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(procs), 5).items()})
    pipe.unet.finalize()
    emb = torch.randn(1, TINY.pooled_embed_dim, generator=torch.Generator("cpu").manual_seed(5)).half()
    kw = dict(pil_image=None, clip_image_embeds=emb, prompt="lions", negative_prompt="blurry", scale=0.8, num_samples=2,
              num_inference_steps=3, seed=[42, 43], height=256, width=256)
    images = ip.generate(output_type="pil", **kw)
    lat = ip.generate(output_type="latent", **kw)
    want = postprocess(pipe.vae.decode(lat), "pil")
    assert len(images) == 2 and all(isinstance(im, Image.Image) and im.size == (256, 256) for im in images)
    for a, b in zip(images, want):
        assert a.tobytes() == b.tobytes()
