"""Host logic of tools/bench_inpaint9.py: conv_in's algorithmic bytes and FLOPs as patch matrix + GEMM."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_inpaint9 import conv_in_cost  # noqa: E402


def test_conv_in_cost_hand_count():
    # 1024^2, CFG batch 2: M = 2 * 128 * 128 rows of the patch matrix
    m = 2 * 128 * 128
    four, nine = conv_in_cost(2, 128, 128, 4, 64), conv_in_cost(2, 128, 128, 9, 128)
    assert four["im2col_bytes"] == 2 * (m * 4 + m * 64) and nine["im2col_bytes"] == 2 * (m * 9 + m * 128)
    assert nine["gemm_bytes"] == 2 * (m * 128 + 320 * 128 + 320 + m * 320)
    # the patch matrix doubles from 4.2 to 8.4 MB, the GEMM from 1.3 to 2.7 GFLOP per step
    assert round(2 * m * 64 / 1e6, 1) == 4.2 and round(2 * m * 128 / 1e6, 1) == 8.4
    assert round(four["gemm_flop"] / 1e9, 1) == 1.3 and round(nine["gemm_flop"] / 1e9, 1) == 2.7
