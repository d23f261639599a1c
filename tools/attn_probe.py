"""A/B timing of the KV-split self-attention plan (graph-timed).  Steering only, not bench values."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from imagharmony_b200 import ops  # noqa: E402
from tools.microbench import timeit, r  # noqa: E402


def main():
    for (B, H, N) in [(2, 20, 1024), (2, 10, 4096), (4, 20, 1024), (8, 20, 1024), (2, 20, 576), (2, 10, 2304)]:
        C = H * 64
        qkv = r(B * N, 3 * C)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        fl = 4.0 * B * H * N * N * 64
        t0 = timeit(lambda: ops.attention(q, k, v, B, H, N, N, kv_split=False))
        t1 = timeit(lambda: ops.attention(q, k, v, B, H, N, N, kv_split=True))
        print(f"self-attn B{B} H{H} N{N}: whole {t0*1e6:.1f} us ({fl/t0/1e12:.0f} TF/s) -> kv-split {t1*1e6:.1f} us "
              f"({fl/t1/1e12:.0f} TF/s)", flush=True)


if __name__ == "__main__":
    main()
