"""SDXL refiner timing on one GPU: the refiner's denoise step and the base -> refiner ensemble of experts.

    python tools/bench_refiner.py [--steps 50] [--handoff 0.8] [--warmup 1] [--res 1024] [--images 1]

Prints one JSON line and writes it to tools_out/bench_refiner.json.  Weights are random-init (SDXL-base UNet with its
IP processors, SDXL refiner UNet), inputs are synthetic N(0, 1) embeddings (77 + 4 tokens for the base, 77 for the
refiner), guidance 5.0 (CFG: UNet batch 2 x images).
  refiner_step : DenoiseEngine.run of the refiner over the whole `steps` schedule (graph replays), CUDA events around
                 the call after a warm-up call; ms per step, steps/s, and the algorithmic FLOPs of one refiner forward
                 (unet_flops, from the config) with the rate against the tensor peak bench.py uses
  ensemble_ms  : base over the steps before the handoff (denoising_end) then the refiner from there (denoising_start),
                 against base_only_ms, the base over the whole schedule; host wall time of each after a warm-up, both
                 from pinned host inputs to latents on the host, VAE decode not included
The card's name and power limit are read in the same process and reported with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_img2img import card  # noqa: E402

TEXT_TOKENS = 77


def unet_flops(cfg, H: int, W: int, batch: int = 1, text_tokens: int = TEXT_TOKENS) -> int:
    """Algorithmic FLOPs (2 per multiply-add) of one UNet forward on [batch, 4, H/8, W/8] latents: every conv
    (conv_in / conv_out, the ResBlocks' two 3x3 convs and 1x1 shortcuts, down- and upsamplers) and every transformer
    block (proj_in / proj_out; self-attention q|k|v, q k^T, P v, out; cross-attention q, k|v of the text tokens, q k^T,
    P v, out; GEGLU and FF-out).  Norms, pointwise ops, the time embeddings and image-prompt tokens are not counted
    (the refiner has none)."""
    def conv(h, w, ci, co, k=3):
        return 2 * h * w * ci * co * k * k

    Lk, D = text_tokens, cfg.cross_attention_dim

    def transformer(h, w, C, depth):
        N = h * w
        blk = (4 * 2 * N * C * C + 2 * 2 * N * N * C             # attn1: q, k, v, out; q k^T, P v
               + 2 * 2 * N * C * C + 2 * 2 * Lk * D * C           # attn2: q, out; k, v of the encoder tokens
               + 2 * 2 * N * Lk * C                               # attn2: q k^T, P v
               + 2 * N * C * 8 * C + 2 * N * 4 * C * C)           # GEGLU (C -> 2 x 4C), FF-out (4C -> C)
        return 2 * 2 * N * C * C + depth * blk if depth else 0

    def resnet(h, w, ci, co):
        return conv(h, w, ci, co) + conv(h, w, co, co) + (conv(h, w, ci, co, 1) if ci != co else 0)

    boc, tl = cfg.block_out_channels, cfg.transformer_layers_per_block
    h, w = H // 8, W // 8
    f = conv(h, w, cfg.in_channels, boc[0])
    skips, ch = [boc[0]], boc[0]
    for i, co in enumerate(boc):
        for j in range(cfg.layers_per_block):
            f += resnet(h, w, ch if j == 0 else co, co) + transformer(h, w, co, tl[i])
            skips.append(co)
        ch = co
        if i < len(boc) - 1:
            h, w = h // 2, w // 2
            f += conv(h, w, co, co)
            skips.append(co)
    f += 2 * resnet(h, w, ch, ch) + transformer(h, w, ch, cfg.mid_depth)
    for i, co in enumerate(reversed(boc)):
        depth = tl[len(boc) - 1 - i]
        for j in range(cfg.layers_per_block + 1):
            f += resnet(h, w, ch + skips.pop(), co) + transformer(h, w, co, depth)
            ch = co
        if i < len(boc) - 1:
            h, w = 2 * h, 2 * w
            f += conv(h, w, co, co)
    f += conv(h, w, boc[0], cfg.out_channels)
    return f * batch


def _inputs(cfg, n: int, lat: int, T: int):
    """Pinned synthetic inputs: latents * init_noise_sigma, [n, 77 + ip tokens, D] embeddings, pooled, time ids."""
    from imagharmony_b200.scheduler import EulerDiscreteScheduler
    g = torch.Generator("cpu").manual_seed(1234 + cfg.num_time_ids)
    ins = EulerDiscreteScheduler().set_timesteps(T).init_noise_sigma
    L = TEXT_TOKENS + cfg.num_ip_tokens
    res = lat * 8.0
    ids = [res, res, 0.0, 0.0] + ([res, res] if cfg.num_time_ids == 6 else [6.0])
    neg_ids = ids[:-1] + [2.5] if cfg.num_time_ids == 5 else ids
    t = [(torch.randn((n, 4, lat, lat), generator=g) * ins).half(),
         torch.randn((n, L, cfg.cross_attention_dim), generator=g).half(),
         torch.randn((n, L, cfg.cross_attention_dim), generator=g).half(),
         torch.randn((n, cfg.pooled_embed_dim), generator=g).half(),
         torch.randn((n, cfg.pooled_embed_dim), generator=g).half(),
         torch.tensor([ids] * n), torch.tensor([neg_ids] * n)]
    return [x.pin_memory() for x in t]


def measure(T: int, handoff: float, W: int, res: int, n: int) -> dict:
    import bench
    from imagharmony_b200.config import SDXL_BASE, SDXL_REFINER
    from imagharmony_b200.denoise import DenoiseEngine
    from ip_adapter.custom_pipelines import denoising_start_begin_step
    if not torch.cuda.is_available():
        raise SystemExit("bench_refiner needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    pk = bench.peaks()
    lat = res // 8
    refiner = DenoiseEngine(bench.build_native(SDXL_REFINER, device), use_cuda_graph=True)
    base = DenoiseEngine(bench.build_native(SDXL_BASE, device), use_cuda_graph=True)
    r_in, b_in = _inputs(SDXL_REFINER, n, lat, T), _inputs(SDXL_BASE, n, lat, T)
    k = denoising_start_begin_step(refiner.scheduler.set_timesteps(T).timesteps, refiner.scheduler.num_train_timesteps,
                                   handoff)

    def run(eng, inputs, **kw):
        x, pe, ne, pp, npp, tid, ntid = inputs
        return eng.run(x, pe, ne, pp, npp, tid, T, guidance_scale=5.0, ip_scale=1.0, negative_time_ids=ntid, **kw)

    for _ in range(max(1, W)):
        run(refiner, r_in)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run(refiner, r_in)
    b.record()
    torch.cuda.synchronize()
    step_ms = a.elapsed_time(b) / T
    flop = unet_flops(SDXL_REFINER, res, res, 2 * n)
    rate = flop / (step_ms * 1e-3) / 1e12
    out = {"card": card(), "res": res, "images": n, "steps": T, "handoff": handoff, "base_steps": k,
           "refiner_steps": T - k,
           "refiner_step": {"workload": f"SDXL refiner UNet (random init), {n} image(s), CFG batch {2 * n}, {res}^2, "
                                        "77 text tokens, graph replays",
                            "ms_per_step": step_ms, "steps_per_s": 1e3 / step_ms, "flop_algorithmic": flop,
                            "tflops_achieved": rate, "frac_of_tensor_peak": rate / pk["tflops_sustained"],
                            "peak_source": pk["source"]}}

    def ensemble():
        mid = run(base, b_in, num_loop_steps=k) if k > 0 else b_in[0]
        x = run(refiner, [mid] + r_in[1:], begin_step=k) if k < T else mid
        return x.to("cpu")

    def base_only():
        return run(base, b_in).to("cpu")

    for name, fn in (("ensemble_ms", ensemble), ("base_only_ms", base_only)):
        for _ in range(max(1, W)):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = fn()
        torch.cuda.synchronize()
        out[name] = (time.perf_counter() - t0) * 1e3
        if not torch.isfinite(host.float()).all():
            raise RuntimeError(f"non-finite latents ({name})")
    out["note"] = ("ensemble: base steps [0, base_steps) then refiner steps [base_steps, steps) on one schedule; "
                   "latents from pinned host memory to the host, VAE decode not included")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--handoff", type=float, default=0.8)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--images", type=int, default=1)
    args = ap.parse_args()
    line = measure(max(1, args.steps), args.handoff, args.warmup, args.res, args.images)
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_refiner.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
