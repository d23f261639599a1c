"""Host logic of tools/bench_controlnet.py: the skip shapes, the injection kernel's algorithmic bytes and the
conditioning embedding's FLOPs, against hand counts."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_controlnet import embedding_flop, injection_bytes, skip_shapes  # noqa: E402


def test_skip_shapes_sdxl_1024():
    sh = skip_shapes((320, 640, 1280), 2, 128)
    assert sh == [(128, 128, 320)] * 3 + [(64, 64, 320)] + [(64, 64, 640)] * 2 + [(32, 32, 640)] \
        + [(32, 32, 1280)] * 3


def test_injection_bytes_hand_count():
    sh = skip_shapes((320, 640, 1280), 2, 128)
    per_image = 3 * 128 * 128 * 320 + 64 * 64 * 320 + 2 * 64 * 64 * 640 + 32 * 32 * 640 + 3 * 32 * 32 * 1280
    full = injection_bytes(sh, 2, 2)
    assert full["skip_bytes"] == 2 * 2 * per_image
    assert round(full["skip_bytes"] / 1e6, 1) == 107.5                    # the skips of a 1024^2 CFG step
    assert full["algorithmic_bytes"] == 3 * full["skip_bytes"]            # read twice (skip, residual), written once
    guess = injection_bytes(sh, 2, 1)                                      # guess mode: the conditional half only
    assert guess["skip_bytes"] == full["skip_bytes"] and 2 * guess["algorithmic_bytes"] == full["algorithmic_bytes"]


def test_embedding_flop_hand_count():
    # 1024^2 image: conv_in 3->16 at 1024, 16->16 at 1024, 16->32 s2 at 512, 32->32 at 512, 32->96 s2 at 256,
    # 96->96 at 256, 96->256 s2 at 128, conv_out 256->320 at 128
    px = {1024: 1024 * 1024, 512: 512 * 512, 256: 256 * 256, 128: 128 * 128}
    want = 18 * (px[1024] * (16 * 3 + 16 * 16) + px[512] * (32 * 16 + 32 * 32) + px[256] * (96 * 32 + 96 * 96)
                 + px[128] * (256 * 96 + 320 * 256))
    assert embedding_flop(1024, 1024, (16, 32, 96, 256), 320) == want
    assert round(want / 1e9, 1) == 58.9
