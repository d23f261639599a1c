"""Host logic of tools/bench_multi_controlnet.py: the fused injection kernel's algorithmic bytes against hand counts."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_controlnet import skip_shapes  # noqa: E402
from tools.bench_multi_controlnet import multi_injection_bytes  # noqa: E402


def test_multi_injection_bytes_hand_count():
    sh = skip_shapes((320, 640, 1280), 2, 128)
    per_image = 3 * 128 * 128 * 320 + 64 * 64 * 320 + 2 * 64 * 64 * 640 + 32 * 32 * 640 + 3 * 32 * 32 * 1280
    touched = 2 * 2 * per_image                                  # fp16 skips of a 1024^2 CFG step
    for k in (1, 2, 3):
        got = multi_injection_bytes(sh, 2, 2, k)
        assert got["touched_skip_bytes"] == got["skip_bytes"] == touched
        assert got["algorithmic_bytes"] == (2 + k) * touched      # skips read + written, k residuals read
    assert round(multi_injection_bytes(sh, 2, 2, 2)["algorithmic_bytes"] / 1e6) == 430
    guess = multi_injection_bytes(sh, 2, 1, 2)                    # guess mode: the conditional half only
    assert guess["skip_bytes"] == touched and 2 * guess["algorithmic_bytes"] == 4 * touched
