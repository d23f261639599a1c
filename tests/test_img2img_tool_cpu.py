"""Host logic of tools/bench_img2img.py: the VAE-encoder FLOP count it reports the achieved rate with."""
import os
import sys


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_img2img import vae_encoder_flops  # noqa: E402


def test_vae_encoder_flops_tiny_hand_sum():
    from imagharmony_b200.config import TINY_VAE           # (64, 64, 128, 128), one ResBlock per level, 4 latents
    hand = (2 * 64 * 64 * 3 * 64 * 9                          # conv_in at 64^2
            + 2 * (2 * 64 * 64 * 64 * 64 * 9) + 2 * 32 * 32 * 64 * 64 * 9           # level 0 ResBlock, downsample
            + 2 * (2 * 32 * 32 * 64 * 64 * 9) + 2 * 16 * 16 * 64 * 64 * 9           # level 1
            + 2 * 16 * 16 * 64 * 128 * 9 + 2 * 16 * 16 * 128 * 128 * 9 + 2 * 16 * 16 * 64 * 128
            + 2 * 8 * 8 * 128 * 128 * 9                                              # level 2 (+ shortcut), downsample
            + 2 * (2 * 8 * 8 * 128 * 128 * 9)                                        # level 3
            + 4 * (2 * 8 * 8 * 128 * 128 * 9)                                        # mid ResBlocks
            + 4 * 2 * 64 * 128 * 128 + 2 * 2 * 64 * 64 * 128                         # mid attention
            + 2 * 8 * 8 * 128 * 8 * 9 + 2 * 8 * 8 * 8 * 8)                           # conv_out, quant_conv
    assert vae_encoder_flops(TINY_VAE, 64, 64) == hand
    assert vae_encoder_flops(TINY_VAE, 64, 64, batch=3) == 3 * hand


def test_vae_encoder_flops_scale_with_area():
    from imagharmony_b200.config import SDXL_VAE
    f512, f1024 = vae_encoder_flops(SDXL_VAE, 512, 512), vae_encoder_flops(SDXL_VAE, 1024, 1024)
    attn = lambda n: 2 * 2 * n * n * 512                      # noqa: E731  (the only term that is not linear in area)
    assert f1024 - attn(128 * 128) == 4 * (f512 - attn(64 * 64))
    assert 4.0 < f1024 / f512 < 4.5
    assert 4.0e12 < f1024 < 6.0e12                           # about 4.9 TFLOP for the SDXL encoder at 1024^2
