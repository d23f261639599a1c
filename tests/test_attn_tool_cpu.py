"""Host logic of tools/bench_attn.py: the attention FLOP count, the shape table and the spread summary."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_attn import SHAPES, attn_flops, spread  # noqa: E402


def test_attn_flops_hand_count():
    # QK^T and PV: 2 * Nq * Nk * 64 each per (batch, head)
    assert attn_flops(1, 1, 128, 128) == 2 * (2 * 128 * 128 * 64)
    # the 1024^2 UNet shapes (DESIGN.md): 85.9 GFLOP per 64^2-token layer, 10.7 per 32^2-token layer
    assert attn_flops(2, 10, 4096, 4096) == 85_899_345_920
    assert attn_flops(2, 20, 1024, 1024) == 10_737_418_240
    assert attn_flops(1, 3, 2000, 1500) == 4 * 3 * 2000 * 1500 * 64


def test_shapes_cover_both_1024_levels_and_a_ragged_one():
    dims = {s[1:] for s in SHAPES}
    assert {(2, 10, 4096, 4096), (2, 20, 1024, 1024), (2, 10, 1024, 1024), (2, 20, 256, 256)} <= dims
    assert any(nq % 128 or nk % 128 for _, _, _, nq, nk in SHAPES)
    assert all(nk > 128 for *_, nk in SHAPES)   # every shape takes the multi-block path the tool compares


def test_spread_summary():
    assert spread([3.0, 1.0, 2.0]) == {"median": 2.0, "min": 1.0, "max": 3.0, "spread": 2.0}
