"""Host logic of tools/bench_t2i_adapter.py: the adapter's FLOP and byte counts and the injection's algorithmic bytes,
against hand counts."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_t2i_adapter import adapter_cost, injection_bytes  # noqa: E402


def test_adapter_flop_hand_count_1024():
    # 64^2 grid: conv_in 768 -> 320 (3x3); block 0: 2 x (3x3 + 1x1) at 320; block 1: 1x1 320 -> 640, 2 x (3x3 + 1x1) at
    # 640; at 32^2: 1x1 640 -> 1280 after the pool, 2 x (3x3 + 1x1) at 1280; block 3: 2 x (3x3 + 1x1) at 1280
    p, q = 64 * 64, 32 * 32
    conv_in = 2 * p * 9 * 768 * 320
    b0 = 2 * 2 * p * 10 * 320 * 320
    b1 = 2 * p * 320 * 640 + 2 * 2 * p * 10 * 640 * 640
    b2 = 2 * q * 640 * 1280 + 2 * 2 * q * 10 * 1280 * 1280
    b3 = 2 * 2 * q * 10 * 1280 * 1280
    assert [round(v / 1e9) for v in (conv_in, b0, b1, b2, b3)] == [18, 17, 69, 69, 67]
    flop, _ = adapter_cost(1024, 1024)
    assert flop == conv_in + b0 + b1 + b2 + b3 and round(flop / 1e9) == 240
    assert adapter_cost(1024, 1024, batch=4)[0] == 4 * flop
    assert adapter_cost(1024, 1024, in_channels=1)[0] == flop - 2 * p * 9 * 512 * 320


def test_adapter_bytes_hand_count_1024():
    p, q = 64 * 64, 32 * 32

    def conv(P, ci, co, k):
        return 2 * (P * ci + P * co + k * k * ci * co + co)
    want = 2 * 2 * 3 * 1024 * 1024 + conv(p, 768, 320, 3)
    want += 2 * (conv(p, 320, 320, 3) + conv(p, 320, 320, 1) + 2 * p * 320)
    want += conv(p, 320, 640, 1) + 2 * (conv(p, 640, 640, 3) + conv(p, 640, 640, 1) + 2 * p * 640)
    want += 2 * (p * 640 + q * 640) + conv(q, 640, 1280, 1)
    want += 4 * (conv(q, 1280, 1280, 3) + conv(q, 1280, 1280, 1) + 2 * q * 1280)
    assert adapter_cost(1024, 1024)[1] == want


def test_injection_bytes_hand_count():
    elems = 64 * 64 * 320 + 64 * 64 * 640 + 2 * 32 * 32 * 1280
    assert elems == 6553600                                   # 6.6 M per image: 13 M with the CFG halves
    assert injection_bytes(1024, 1024) == 3 * 2 * 2 * elems   # skip read + feature read + skip write, 2 halves
    assert round(injection_bytes(1024, 1024) / 1e6) == 79
    assert injection_bytes(1024, 1024, cfg=False) * 2 == injection_bytes(1024, 1024)
