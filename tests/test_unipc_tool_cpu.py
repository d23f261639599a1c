"""Host logic of tools/bench_unipc.py: the UniPC step kernel's algorithmic byte count."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_dpm import dpm_step_bytes  # noqa: E402
from tools.bench_unipc import E2E, unipc_step_bytes  # noqa: E402


def test_unipc_step_bytes_hand_count():
    # CFG, n = 1, 128 x 128 latents: reads pred 2x4, latents 4, last_sample 4, prev x0 4, prev x0_2 4 planes;
    # writes latents 4, last_sample 4, prev x0 4, prev x0_2 4, model_in 2x4
    plane = 128 * 128 * 2
    assert unipc_step_bytes(1, 4, 128, 128, True) == (8 + 4 * 4 + 4 * 4 + 8) * plane == 1572864
    assert unipc_step_bytes(1, 4, 128, 128, False) == (4 + 4 * 4 + 4 * 4 + 4) * plane
    assert unipc_step_bytes(3, 4, 64, 32, True) == 3 * unipc_step_bytes(1, 4, 64, 32, True)
    # two more history tensors than DPM-Solver++, each read and written
    assert unipc_step_bytes(1, 4, 128, 128, True) - dpm_step_bytes(1, 4, 128, 128, True) == 2 * 2 * 4 * plane


def test_end_to_end_configurations():
    assert E2E == (("unipc", 10), ("dpmpp_2m_karras", 20), ("dpmpp_2m_karras", 25))
