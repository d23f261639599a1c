"""Self-attention kernel A/B: the persistent warp-specialised kernel (ih_attention_set_kernel(0), the default) against
the two-CTA-per-SM kernel (1) on the multi-block shapes of the SDXL UNet.

  python tools/bench_attn.py [--rounds 7] [--launches 50] [--out FILE]

For every shape both kernels run on the same fused q|k|v view (row stride 3C, as the UNet calls them), alternated
over `rounds` rounds of `launches` back-to-back launches each, timed with CUDA events after a warm-up.  The KV-split
plan is on (as in the UNet).  Reported per kernel: median and spread (max - min) of the per-launch time over the
rounds, TFLOP/s from 4 B H Nq Nk 64, and that rate as a fraction of the 989 TFLOP/s dense FP16 data-sheet figure of
the H100 SXM (a data-sheet figure, not a reached one).  Each shape also checks that the two kernels' outputs are
torch.equal with the split withheld.  The card's name, power limit and maximum SM clock are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATASHEET_TFLOPS = 989.0    # H100 SXM, dense FP16 / BF16

# (label, B, H, Nq, Nk): CFG pair (B = 2) at 1024^2 and 512^2, and one ragged shape
SHAPES = [
    ("1024^2 64^2 tokens", 2, 10, 4096, 4096),
    ("1024^2 32^2 tokens", 2, 20, 1024, 1024),
    ("512^2 32^2 tokens", 2, 10, 1024, 1024),
    ("512^2 16^2 tokens", 2, 20, 256, 256),
    ("ragged", 1, 3, 2000, 1500),
]


def attn_flops(B: int, H: int, Nq: int, Nk: int) -> float:
    """Algorithmic FLOPs of softmax(q k^T) v at head dim 64: two GEMMs of 2 Nq Nk 64 each per (batch, head)."""
    return 4.0 * B * H * Nq * Nk * 64


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs)}


def measure(rounds: int, launches: int) -> dict:
    import torch
    from imagharmony_b200 import _lib, ops
    from tools.bench_img2img import card
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn needs a GPU")
    lib = _lib.load()
    torch.cuda.set_device(0)
    out = {"card": card(), "rounds": rounds, "launches": launches, "datasheet_tflops": DATASHEET_TFLOPS, "shapes": []}
    g = torch.Generator("cpu").manual_seed(0)
    for label, B, H, Nq, Nk in SHAPES:
        C = H * 64
        qkv_q = torch.randn(B * Nq, 3 * C, generator=g).half().cuda()
        qkv_k = qkv_q if Nq == Nk else torch.randn(B * Nk, 3 * C, generator=g).half().cuda()
        q, k, v = qkv_q[:, :C], qkv_k[:, C:2 * C], qkv_k[:, 2 * C:]
        res = torch.empty(B * Nq, C, dtype=torch.float16, device="cuda")
        whole = {}
        for kern in (0, 1):
            lib.ih_attention_set_kernel(kern)
            whole[kern] = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=False)
            for _ in range(5):
                ops.attention(q, k, v, B, H, Nq, Nk, out=res)
        torch.cuda.synchronize()
        times = {0: [], 1: []}
        for _ in range(rounds):
            for kern in (1, 0):
                lib.ih_attention_set_kernel(kern)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(launches):
                    ops.attention(q, k, v, B, H, Nq, Nk, out=res)
                e1.record()
                e1.synchronize()
                times[kern].append(e0.elapsed_time(e1) / launches)
        lib.ih_attention_set_kernel(0)
        fl = attn_flops(B, H, Nq, Nk)
        row = {"shape": label, "B": B, "H": H, "Nq": Nq, "Nk": Nk, "gflop": fl / 1e9,
               "equal_whole": bool(torch.equal(whole[0], whole[1]))}
        for kern, name in ((1, "old"), (0, "new")):
            st = spread(times[kern])
            tf = fl / (st["median"] * 1e-3) / 1e12
            row[name] = {"ms": st, "tflops": tf, "frac_of_datasheet": tf / DATASHEET_TFLOPS}
        row["speedup"] = row["old"]["ms"]["median"] / row["new"]["ms"]["median"]
        out["shapes"].append(row)
        print(f"{label:>20}  old {row['old']['ms']['median'] * 1e3:8.1f} us (+-{row['old']['ms']['spread'] * 1e3:.1f}) "
              f"{row['old']['tflops']:5.0f} TF/s | new {row['new']['ms']['median'] * 1e3:8.1f} us "
              f"(+-{row['new']['ms']['spread'] * 1e3:.1f}) {row['new']['tflops']:5.0f} TF/s | x{row['speedup']:.3f} "
              f"| equal {row['equal_whole']}", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    res = measure(a.rounds, a.launches)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
