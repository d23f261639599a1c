"""GPU parity of the native VAE decoder (scope row f1) against the CPU fp32 oracle (oracle/vae_ref.py, [3P] restated,
parity unpinned) with identical fp16-representable random weights, through the C ABI kernels.  Bar: the native fp16
pipeline may not be further from the fp32 oracle than 2x the same oracle evaluated in torch fp16 on the GPU."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _models(cfg, seed):
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle.vae_ref import VAEDecoderRef
    with torch.device("meta"):
        shapes = shapes_of(VAEDecoderRef(cfg))
    sd = random_state_dict(shapes, seed)
    native = AutoencoderKLDecoder.from_state_dict(cfg, sd, device="cuda")
    ref32 = VAEDecoderRef(cfg)
    ref32.load_state_dict({k: v.float() for k, v in sd.items()})
    eager16 = VAEDecoderRef(cfg)
    eager16.load_state_dict({k: v.float() for k, v in sd.items()})
    return native, ref32.eval(), eager16.half().cuda().eval()


def _check(cfg, seed, B, lat):
    native, ref32, eager16 = _models(cfg, seed)
    g = torch.Generator("cpu").manual_seed(seed + 1)
    z = (torch.randn(B, 4, lat, lat, generator=g) * cfg.scaling_factor * 2).half()     # latent-scale inputs
    with torch.no_grad():
        r = ref32.decode(z.float())
        e = eager16.decode(z.cuda()).float().cpu()
        o = native.decode(z.cuda()).float().cpu()
    torch.cuda.synchronize()
    e_nat, e_eag, mx = (o - r).abs().max().item(), (e - r).abs().max().item(), r.abs().max().item()
    rms = ((o - r).pow(2).mean().sqrt() / r.pow(2).mean().sqrt()).item()
    print(f"[vae {cfg.block_out_channels} B{B} {lat}x{lat}] native err {e_nat:.3e}  eager-fp16 err {e_eag:.3e}  "
          f"max|ref| {mx:.3e}  rel-RMS {rms:.3e}")
    assert o.shape == (B, 3, 8 * lat, 8 * lat) and torch.isfinite(o).all()
    assert e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
    return o, r


def test_softmax_rows_kernel():
    from imagharmony_b200 import ops
    for rows, cols in [(64, 1024), (33, 4096), (16, 16384), (8, 32768), (5, 200)]:
        g = torch.Generator("cpu").manual_seed(rows)
        x = (torch.randn(rows, cols, generator=g) * 3).half().cuda()
        big = torch.zeros(rows, cols + 64, dtype=torch.float16, device="cuda")
        view = big[:, :cols]
        view.copy_(x)
        ops.softmax_rows_masked_(view, cols)                       # strided rows, in place, every column valid
        ref = torch.softmax(x.float(), dim=-1)
        assert torch.allclose(view.float(), ref, rtol=2e-3, atol=1e-6), (view.float() - ref).abs().max()
        assert (big[:, cols:] == 0).all()


def test_vae_decoder_tiny_matches_oracle():
    from imagharmony_b200.config import TINY_VAE
    _check(TINY_VAE, seed=5, B=2, lat=8)
    _check(TINY_VAE, seed=6, B=1, lat=12)        # 144 mid-block tokens: not a multiple of 128


def test_vae_decoder_sdxl_256_matches_oracle_and_postprocess():
    """The full SDXL VAE decoder architecture (49.5 M parameters) on a 32x32 latent -> 256x256 image, and the uint8
    image after postprocess within one grey level of the oracle's."""
    from imagharmony_b200.config import SDXL_VAE
    from imagharmony_b200.vae import postprocess
    from oracle.vae_ref import postprocess_ref
    o, r = _check(SDXL_VAE, seed=7, B=1, lat=32)
    u8 = np.asarray(postprocess(o, "pil")[0]).astype(np.int32)
    r8 = (postprocess_ref(r)[0] * 255).round().astype(np.int32)
    assert u8.shape == (256, 256, 3)
    assert np.abs(u8 - r8).max() <= 1, np.abs(u8 - r8).max()


def test_vae_tiled_decode_matches_oracle():
    """enable_vae_tiling (test.py:73): overlapping 8x8-latent tiles of the miniature VAE incl. ragged edge tiles (token
    counts that are not multiples of 8 -> padded keys with -inf scores) against the oracle's tiled_decode."""
    from imagharmony_b200.config import TINY_VAE
    from oracle.vae_ref import tiled_decode_ref
    native, ref32, _ = _models(TINY_VAE, seed=9)
    native.use_tiling = True
    z = (torch.randn(1, 4, 14, 11, generator=torch.Generator("cpu").manual_seed(3)) * TINY_VAE.scaling_factor * 2).half()
    with torch.no_grad():
        r = tiled_decode_ref(ref32, z.float())
        o = native.decode(z.cuda()).float().cpu()
    torch.cuda.synchronize()
    err, mx = (o - r).abs().max().item(), r.abs().max().item()
    print(f"[vae tiled] max|err| {err:.3e} max|ref| {mx:.3e}")
    assert o.shape == r.shape and torch.isfinite(o).all()
    assert err <= 1e-2 * mx, (err, mx)


def test_softmax_rows_masked_kernel():
    from imagharmony_b200 import ops
    for rows, cols, valid in [(64, 1024, 1000), (7, 168, 165), (16, 16384, 16384)]:
        x = (torch.randn(rows, cols, generator=torch.Generator("cpu").manual_seed(rows)) * 3).half().cuda()
        ref = torch.zeros(rows, cols)
        ref[:, :valid] = torch.softmax(x[:, :valid].float().cpu(), dim=-1)
        ops.softmax_rows_masked_(x, valid)
        assert torch.allclose(x.float().cpu(), ref, rtol=2e-3, atol=1e-6) and (x[:, valid:] == 0).all()


def test_vae_scaled_stream_survives_fp16_overflow():
    """The reference upcasts the SDXL VAE to fp32 because its activations overflow fp16 (custom_pipelines.py:366-371).
    A decoder whose residual stream reaches ~1e5 (conv_in scaled up 4000x, latents 8x the usual range): the plain fp16 pipeline (stream_scale 1, and
    the torch fp16 oracle) produces non-finite pixels, the scaled-stream pipeline (default 2^-7) matches the fp32 oracle."""
    from imagharmony_b200.config import TINY_VAE as cfg
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle.vae_ref import VAEDecoderRef
    with torch.device("meta"):
        shapes = shapes_of(VAEDecoderRef(cfg))
    sd = {k: v.float() for k, v in random_state_dict(shapes, 11).items()}
    for k in ("decoder.conv_in.weight", "decoder.conv_in.bias"):
        sd[k] = (sd[k] * 4000.0).half().float()              # stays fp16-representable, so does the folded conv_in weight
    ref32 = VAEDecoderRef(cfg)
    ref32.load_state_dict(sd)
    z = (torch.randn(2, 4, 16, 16, generator=torch.Generator("cpu").manual_seed(12)) * cfg.scaling_factor * 16).half()
    with torch.no_grad():
        r = ref32.eval().decode(z.float())
        stream = ref32.decoder.conv_in(ref32.post_quant_conv(z.float() / cfg.scaling_factor))
    assert stream.abs().max() > 65504, "the test model must overflow fp16"
    native = AutoencoderKLDecoder.from_state_dict(cfg, sd, device="cuda")
    assert native.stream_scale == 2.0 ** -7
    o = native.decode(z.cuda()).float().cpu()
    plain = AutoencoderKLDecoder.from_state_dict(cfg, sd, device="cuda", stream_scale=1.0).decode(z.cuda()).float().cpu()
    torch.cuda.synchronize()
    err, mx = (o - r).abs().max().item(), r.abs().max().item()
    print(f"[vae scaled stream] stream max {stream.abs().max().item():.3e}: scaled max|err| {err:.3e} (max|ref| {mx:.3e}); "
          f"plain fp16 finite: {bool(torch.isfinite(plain).all())}")
    assert torch.isfinite(o).all() and err <= 1e-2 * mx, (err, mx)
    assert not torch.isfinite(plain).all(), "without the scaled stream this model overflows fp16"
