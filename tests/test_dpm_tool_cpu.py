"""Host logic of tools/bench_dpm.py: the step kernels' algorithmic byte counts and the spread summary."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_dpm import dpm_step_bytes, euler_step_bytes, spread  # noqa: E402


def test_dpm_step_bytes_hand_count():
    # CFG, n = 1, 128 x 128 latents: reads pred 2x4, latents 4, prev x0 4 planes; writes latents 4, x0 4, model_in 2x4
    plane = 128 * 128 * 2
    assert dpm_step_bytes(1, 4, 128, 128, True) == (8 + 4 + 4 + 4 + 4 + 8) * plane == 1048576   # 1 MB per 1024^2 image
    assert dpm_step_bytes(1, 4, 128, 128, False) == (4 + 4 + 4 + 4 + 4 + 4) * plane
    assert dpm_step_bytes(3, 4, 64, 32, True) == 3 * dpm_step_bytes(1, 4, 64, 32, True)
    # the Euler kernel: no x0 history
    assert euler_step_bytes(1, 4, 128, 128, True) == (8 + 4 + 4 + 8) * plane


def test_spread_summary():
    assert spread([3.0, 1.0, 2.0]) == {"median": 2.0, "min": 1.0, "max": 3.0, "spread": 2.0}
