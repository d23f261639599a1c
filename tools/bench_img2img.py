"""Image-to-image timing on one GPU: the SDXL VAE encoder and one img2img call on the bench workload.

    python tools/bench_img2img.py [--strength 0.6] [--steps 20] [--warmup 3] [--res 1024] [--images 1]

Prints one JSON line and writes it to tools_out/bench_img2img.json.  Weights are random-init SDXL-base (UNet, IP
processors, VAE encoder), inputs are bench.py's synthetic embeddings.
  vae_encode : AutoencoderKLEncoder.encode_moments_nhwc on [images, 3, res, res] in [-1, 1], CUDA events over 5 calls
               after 2 warm-up calls; the encoder's algorithmic FLOPs (vae_encoder_flops, from shapes) and the rate
               against the tensor peak bench.py uses (data sheet unless MEASURED_PEAKS.json exists)
  steps_kept : denoise steps a `strength` leaves of the `steps`-step schedule (diffusers get_timesteps)
  e2e_ms     : one call after a warm-up call: encode + eps / noise draws + ops.vae_posterior_noise + DenoiseEngine.run
               over the truncated schedule (graph replays) + D2H of the latents; VAE decode is not included
The card's name and power limit are read in the same process and reported with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def vae_encoder_flops(cfg, H: int, W: int, batch: int = 1) -> int:
    """Algorithmic FLOPs (2 per multiply-add) of the [3P] AutoencoderKL encoder + quant_conv on [batch, 3, H, W]:
    every conv, the mid-block attention's four projections and its two N x N products; norms and pointwise ops are
    not counted."""
    def conv(h, w, ci, co, k):
        return 2 * h * w * ci * co * k * k
    ch = cfg.block_out_channels
    h, w = H, W
    f = conv(h, w, cfg.out_channels, ch[0], 3)
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg.layers_per_block):
            ci = prev if j == 0 else c
            f += conv(h, w, ci, c, 3) + conv(h, w, c, c, 3) + (conv(h, w, ci, c, 1) if ci != c else 0)
        prev = c
        if i < len(ch) - 1:                               # Downsample2D: pad (0, 1, 0, 1), 3x3 stride 2
            h, w = h // 2, w // 2
            f += conv(h, w, c, c, 3)
    C, N, z = ch[-1], h * w, 2 * cfg.latent_channels
    f += 4 * conv(h, w, C, C, 3)                          # mid block: two ResBlocks
    f += 4 * 2 * N * C * C + 2 * 2 * N * N * C            # attention: q, k, v, out projections; q k^T and P v
    f += conv(h, w, C, z, 3) + conv(h, w, z, z, 1)        # conv_out, quant_conv
    return f * batch


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception as ex:  # pragma: no cover
        return f"unknown ({ex})"


def measure(strength: float, K: int, W: int, res: int, n: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE, SDXL_VAE
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    if not torch.cuda.is_available():
        raise SystemExit("bench_img2img needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    pk = bench.peaks()
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLEncoder(SDXL_VAE))
    venc = AutoencoderKLEncoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 23, device=str(device)), device=device)
    image = (torch.rand((n, 3, res, res), generator=torch.Generator("cpu").manual_seed(5)) * 2 - 1).half().to(device)
    for _ in range(2):                                                  # warm-up: TMA descriptors, workspaces
        venc.encode_moments_nhwc(image)
    torch.cuda.synchronize()
    reps = 5
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        venc.encode_moments_nhwc(image)
    b.record()
    torch.cuda.synchronize()
    enc_ms = a.elapsed_time(b) / reps
    flop = vae_encoder_flops(SDXL_VAE, res, res, n)
    rate = flop / (enc_ms * 1e-3) / 1e12

    eng = DenoiseEngine(bench.build_native(SDXL_BASE, device), use_cuda_graph=True)
    lat = res // 8
    run_args = [t.pin_memory() for t in bench.synth_inputs(SDXL_BASE, n, lat, K, 0)]
    t_start = eng.scheduler.img2img_begin_index(K, strength)
    out = {"card": card(), "strength": strength, "steps_kept": K - t_start, "of_steps": K,
           "vae_encode": {"workload": f"SDXL VAE encoder + quant_conv, {n} x 3 x {res} x {res}, scaled fp16 stream",
                          "ms": enc_ms, "flop_algorithmic": flop, "tflops_achieved": rate,
                          "frac_of_tensor_peak": rate / pk["tflops_sustained"], "peak_source": pk["source"]}}
    if K - t_start < 1:
        out["e2e_ms"] = None
        return out
    sigma = float(eng.scheduler.set_timesteps(K).sigmas[t_start])
    g = torch.Generator(device).manual_seed(7)

    def call():
        moments = venc.encode_moments_nhwc(image)
        eps = torch.randn((n, 4, lat, lat), generator=g, device=device, dtype=torch.float32)
        noise = torch.randn((n, 4, lat, lat), generator=g, device=device, dtype=torch.float16)
        x = ops.vae_posterior_noise(moments, eps, noise, 4, SDXL_VAE.scaling_factor, sigma)
        return eng.run(x, *run_args[1:6], K, guidance_scale=5.0, ip_scale=1.0, begin_step=t_start).to("cpu")
    for _ in range(max(1, W)):
        call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = call()
    torch.cuda.synchronize()
    out["e2e_ms"] = (time.perf_counter() - t0) * 1e3
    out["e2e_note"] = ("encode + posterior/noise kernel + truncated denoise loop (graph replays) + D2H of the latents; "
                       "embeddings from pinned host memory, VAE decode not included")
    if not torch.isfinite(host.float()).all():
        raise RuntimeError("non-finite img2img latents")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strength", type=float, default=0.6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--images", type=int, default=1)
    args = ap.parse_args()
    line = measure(args.strength, max(1, args.steps), args.warmup, args.res, args.images)
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_img2img.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
