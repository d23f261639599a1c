"""Full SDXL VAE decoder against the tiny autoencoder (TAESD-XL) decoder on one GPU.

    python tools/bench_taesd.py [--warmup 2] [--iters 5] [--batches 1 4 8] [--out tools_out]

For every SDXL resolution bucket (1024^2, 1152x896, 1216x832, 1344x768, 1536x640 and their transposes) and batch it
times `decode` of both decoders (random-init weights of the real architectures) with CUDA events after `warmup`
untimed calls, the median of `iters` timed calls.  With each decode it reports the FLOPs and bytes computed from the
shapes here (kl_cost / tiny_cost), the achieved TFLOP/s, and which bound (compute or HBM bandwidth at the H100 SXM
data-sheet rates) is the larger, i.e. limits the least time the decode could take.  Then the PNS judge of bench.py
(ViT-bigG/14 + bigG text towers) scores 4 candidates of 1024^2 with each decoder: time per candidate.  The card's name,
power limit and max SM clock are read in the same process and printed with the numbers.  One JSON line per case;
all lines also go to <out>/bench_taesd.json.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BUCKETS = [(1024, 1024), (1152, 896), (1216, 832), (1344, 768), (1536, 640),
           (896, 1152), (832, 1216), (768, 1344), (640, 1536)]          # (height, width)
PEAK_FLOPS = 989e12      # H100 SXM data sheet, dense FP16 tensor core
PEAK_BYTES = 3.35e12     # H100 SXM data sheet, HBM3


def _conv(P: int, ci: int, co: int, k: int = 3):
    """(FLOPs, bytes) of a k x k conv over P output pixels (stride 1, fp16): input and output once, the weight once."""
    return 2 * P * k * k * ci * co, 2 * (P * ci + P * co + k * k * ci * co + co)


def kl_cost(cfg, H: int, W: int, batch: int = 1):
    """(FLOPs, bytes) of one AutoencoderKL decode (imagharmony_b200.vae): every conv / linear / attention matmul, and
    for bytes the activations each kernel reads and writes once (GroupNorm reads its input twice: statistics, then
    normalise), the attention's fp16 score blocks written by q k^T, read and written by the softmax and read by P V,
    plus every weight once.  Elementwise glue on the 4-channel latent is left out."""
    h, w = H // 8, W // 8
    P = h * w
    L = cfg.latent_channels
    f = b = 0

    def add(c):
        nonlocal f, b
        f, b = f + c[0], b + c[1]

    def gn(P, C):
        add((0, 2 * 3 * P * C))

    def resnet(P, ci, co):
        gn(P, ci)
        add(_conv(P, ci, co))
        gn(P, co)
        c = _conv(P, co, co)
        add((c[0], c[1] + 2 * P * co))                          # + the residual read
        if ci != co:
            add(_conv(P, ci, co, k=1))

    ch = cfg.decoder_channels
    add(_conv(P, L, L, k=1))                                    # post_quant_conv
    add(_conv(P, L, ch[0]))                                     # conv_in
    resnet(P, ch[0], ch[0])
    C = ch[0]                                                   # mid-block attention, one head of width C
    gn(P, C)
    add((4 * 2 * P * C * C, 2 * (4 * 2 * P * C + 4 * C * C)))   # q, k, v, out projections
    add((2 * 2 * P * P * C, 2 * 4 * P * P))                     # q k^T, P V; the score matrix through the softmax
    resnet(P, ch[0], ch[0])
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg.layers_per_block + 1):
            resnet(P, prev if j == 0 else c, c)
        prev = c
        if i < len(ch) - 1:
            add((0, 2 * (P * c + 4 * P * c)))                   # nearest 2x upsample
            P *= 4
            add(_conv(P, c, c))
    gn(P, ch[-1])
    add(_conv(P, ch[-1], cfg.out_channels))
    return batch * f, batch * b


def tiny_cost(cfg, H: int, W: int, batch: int = 1):
    """(FLOPs, bytes) of one AutoencoderTiny decode (imagharmony_b200.taesd) as it launches: conv_in as im2col (64-wide
    rows written and read) + GEMM, three convs per block (the third also reads the residual), upsample, the bias-free
    conv after it, conv_out (16 padded channels written) and the gather to 3-channel NCHW.  The tanh clamp (torch
    elementwise ops on the 4-channel latent) is left out."""
    h, w = H // 8, W // 8
    P = h * w
    L, C = cfg.latent_channels, cfg.decoder_block_out_channels[0]
    f, b = 2 * P * 9 * L * C, 2 * (P * L + 2 * P * 64 + 64 * C + C + P * C)
    n = len(cfg.num_decoder_blocks)
    for i, nb in enumerate(cfg.num_decoder_blocks):
        for _ in range(nb):
            for k in range(3):
                c = _conv(P, C, C)
                f, b = f + c[0], b + c[1] + (2 * P * C if k == 2 else 0)
        if i < n - 1:
            b += 2 * (P * C + 4 * P * C)
            P *= 4
            c = _conv(P, C, C)
            f, b = f + c[0], b + c[1] - 2 * C                   # bias-free
    c = _conv(P, C, cfg.out_channels)
    f, b = f + c[0], b + c[1] + 2 * P * (16 - cfg.out_channels) + 2 * P * (16 + cfg.out_channels)
    return batch * f, batch * b


def bound(flops: float, byts: float) -> dict:
    tc, tb = flops / PEAK_FLOPS, byts / PEAK_BYTES
    return {"bound": "compute" if tc >= tb else "bandwidth", "min_ms": max(tc, tb) * 1e3}


def _time_ms(fn, warmup: int, iters: int) -> list:
    import torch
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--out", default=os.path.join(ROOT, "tools_out"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_taesd.py needs a GPU")
    import bench
    from imagharmony_b200.config import SDXL_VAE, TAESDXL
    from imagharmony_b200.taesd import AutoencoderTinyDecoder
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from tools.bench_img2img import card
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda"
    with torch.device("meta"):
        kshapes, tshapes = shapes_of(AutoencoderKLDecoder(SDXL_VAE)), shapes_of(AutoencoderTinyDecoder(TAESDXL))
    kl = AutoencoderKLDecoder.from_state_dict(SDXL_VAE, random_state_dict(kshapes, 33, device=dev), device=dev)
    tiny = AutoencoderTinyDecoder.from_state_dict(TAESDXL, random_state_dict(tshapes, 34, device=dev), device=dev)
    gpu = card()
    rows = []
    for H, W in BUCKETS:
        for B in args.batches:
            z = torch.randn(B, 4, H // 8, W // 8, generator=torch.Generator("cpu").manual_seed(B)).half().to(dev)
            row = {"card": gpu, "height": H, "width": W, "batch": B}
            for name, dec, cost in (("kl", kl, kl_cost(SDXL_VAE, H, W, B)), ("tiny", tiny, tiny_cost(TAESDXL, H, W, B))):
                ts = _time_ms(lambda: dec.decode(z), args.warmup, args.iters)
                ms = statistics.median(ts)
                row.update({f"{name}_ms": ms, f"{name}_spread_ms": max(ts) - min(ts), f"{name}_tflop": cost[0] / 1e12,
                            f"{name}_gbytes": cost[1] / 1e9, f"{name}_tflops": cost[0] / ms / 1e9})
                row.update({f"{name}_{k}": v for k, v in bound(*cost).items()})
            row["speedup"] = row["kl_ms"] / row["tiny_ms"]
            rows.append(row)
            print(json.dumps(row), flush=True)
            del z
            torch.cuda.empty_cache()
    # the PNS judge (bench.py's ClipScorer: bigG towers) on 4 candidates of 1024^2, with each decoder
    scorer = bench.build_clip_judge(dev)
    lat = torch.randn(4, 4, 128, 128, generator=torch.Generator("cpu").manual_seed(7)).half().to(dev)
    judge = {"card": gpu, "judge_candidates": 4, "height": 1024, "width": 1024}
    for name, dec in (("kl", kl), ("tiny", tiny)):
        scorer.decode = dec.decode
        ts = _time_ms(lambda: scorer(lat), args.warmup, args.iters)
        judge[f"judge_{name}_ms_per_candidate"] = statistics.median(ts) / 4
        judge[f"judge_{name}_spread_ms"] = max(ts) - min(ts)
    judge["judge_speedup"] = judge["judge_kl_ms_per_candidate"] / judge["judge_tiny_ms_per_candidate"]
    rows.append(judge)
    print(json.dumps(judge), flush=True)
    with open(os.path.join(args.out, "bench_taesd.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
