"""Host logic of tools/bench_euler_a.py: the ancestral step kernel's algorithmic byte count."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_euler_a import euler_a_step_bytes  # noqa: E402


def test_euler_a_step_bytes_hand_count():
    # CFG, n = 1, 128 x 128 latents: reads pred 2x4, latents 4, noise row 4 planes; writes latents 4, model_in 2x4
    plane = 128 * 128 * 2
    assert euler_a_step_bytes(1, 4, 128, 128, True) == (8 + 4 + 4 + 4 + 8) * plane
    assert euler_a_step_bytes(1, 4, 128, 128, False) == (4 + 4 + 4 + 4 + 4) * plane
    assert euler_a_step_bytes(3, 4, 64, 32, True) == 3 * euler_a_step_bytes(1, 4, 64, 32, True)
