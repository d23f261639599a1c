"""Per-shape A/B of GEMM / conv tile widths at the SDXL UNet shapes (batch 2, 1024^2, and the 512^2 q|k|v): each
launch graph-replayed with the old tile choice (192 or 256 columns) and with the one pick_bn now makes, alternated over
several rounds in one process.  Prints and writes tools_out/bench_tiles.json: median and spread of each side,
algorithmic TFLOP/s, and the card's name and power limit read in the same process.

    python tools/bench_tiles.py [--rounds 7] [--iters 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from imagharmony_b200 import ops  # noqa: E402
from tools.microbench import r, timeit  # noqa: E402

# (label, kind, shape, old tile, new tile); GEMM shape (M, N, K), conv shape (B, H, Cin, Cout, stride)
CASES = [
    ("level-2 to_q/to_out/proj", "gemm", (2048, 1280, 1280), 192, 160),
    ("level-2 FF-out", "gemm", (2048, 1280, 5120), 192, 160),
    ("level-1 to_q/to_out/proj", "gemm", (8192, 640, 640), 192, 160),
    ("level-1 FF-out", "gemm", (8192, 640, 2560), 192, 160),
    ("level-2 q|k|v", "gemm", (2048, 3840, 1280), 256, 160),
    ("level-1 q|k|v", "gemm", (8192, 1920, 640), 256, 192),
    ("512^2 level-1 q|k|v", "gemm", (2048, 1920, 640), 256, 128),
    ("level-2 ResBlock conv", "conv", (2, 32, 1280, 1280, 1), 192, 160),
    ("level-2 ResBlock conv (up, 2560 in)", "conv", (2, 32, 2560, 1280, 1), 192, 160),
    ("level-1 ResBlock conv", "conv", (2, 64, 640, 640, 1), 192, 160),
    ("level-0 ResBlock conv", "conv", (2, 128, 320, 320, 1), 192, 160),
]


def power_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as ex:  # noqa
        return f"nvidia-smi unavailable: {ex}"


def make(kind, shape, tile):
    if kind == "gemm":
        M, N, K = shape
        x, w, b = r(M, K), r(N, K, scale=K ** -0.5), r(N)
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        return (lambda: ops.linear(x, w, b, out=out, tile_n=tile)), 2.0 * M * N * K
    B, H, Cin, Cout, s = shape
    x, w, b = r(B, H, H, Cin), r(Cout, 9 * Cin, scale=(9 * Cin) ** -0.5), r(Cout)
    return (lambda: ops.conv3x3(x, w, b, stride=s, tile_n=tile)), 2.0 * B * (H // s) ** 2 * Cout * 9 * Cin


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiles.py needs a GPU")
    card = torch.cuda.get_device_name(0)
    info = {"device": card, "nvidia_smi": power_info(), "rounds": args.rounds, "iters": args.iters, "cases": []}
    print(json.dumps({k: info[k] for k in ("device", "nvidia_smi")}), flush=True)
    for label, kind, shape, old, new in CASES:
        fo, flops = make(kind, shape, old)
        fn, _ = make(kind, shape, new)
        to, tn = [], []
        for i in range(args.rounds):                # alternate, swapping which side goes first: both sides see the
            for side in ((0, 1) if i % 2 == 0 else (1, 0)):     # same clocks, power state and neighbours
                (to if side == 0 else tn).append(timeit(fo if side == 0 else fn, iters=args.iters) * 1e6)
        mo, mn = statistics.median(to), statistics.median(tn)
        row = {"case": label, "kind": kind, "shape": shape, "old_tile": old, "new_tile": new,
               "old_us_median": mo, "old_us_spread": max(to) - min(to), "new_us_median": mn,
               "new_us_spread": max(tn) - min(tn), "old_tflops": flops / mo * 1e-6, "new_tflops": flops / mn * 1e-6,
               "speedup": mo / mn}
        info["cases"].append(row)
        print(json.dumps(row), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_tiles.json"), "w") as fh:
        json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
