"""Host logic of tools/bench_inpaint.py: the step kernels' algorithmic byte counts and the spread summary."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_inpaint import euler_step_bytes, inpaint_step_bytes, spread  # noqa: E402


def test_inpaint_step_bytes_hand_count():
    # CFG, n = 1, 128 x 128 latents: reads pred 2x4, latents 4, image latents 4, noise 4, mask 1 planes; writes 4 + 2x4
    plane = 128 * 128 * 2
    assert inpaint_step_bytes(1, 4, 128, 128, True) == (8 + 4 + 4 + 4 + 1 + 4 + 8) * plane
    assert inpaint_step_bytes(1, 4, 128, 128, False) == (4 + 4 + 4 + 4 + 1 + 4 + 4) * plane
    assert inpaint_step_bytes(3, 4, 64, 32, True) == 3 * inpaint_step_bytes(1, 4, 64, 32, True)
    # what inpainting adds to a step: image latents, noise and mask, about 0.3 MB per 1024^2 image
    extra = inpaint_step_bytes(1, 4, 128, 128, True) - euler_step_bytes(1, 4, 128, 128, True)
    assert extra == 9 * plane == 294912


def test_spread_summary():
    s = spread([3.0, 1.0, 2.0])
    assert s == {"median": 2.0, "min": 1.0, "max": 3.0, "spread": 2.0}
