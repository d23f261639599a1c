"""9-channel inpainting timing on one GPU: the 9-channel inpaint step graph against the 4-channel text-to-image step
graph, conv_in's patch matrix + GEMM of each, and one 9-channel inpaint call end to end.

    python tools/bench_inpaint9.py [--strength 0.6] [--steps 20] [--res 1024] [--rounds 7] [--replays 10]

Prints one JSON line and writes it to tools_out/bench_inpaint9.json.  Weights are random-init SDXL-base (the 4-channel
UNet, the same architecture with a 9-channel conv_in, IP processors, VAE encoder); inputs are bench.py's synthetic
embeddings; the mask regenerates the middle half of the image.
  step_graph: the captured step graph of each kind (UNet forward + Euler kernel, CFG, n = 1) replayed `replays` times
              between CUDA events, the two kinds alternated over `rounds` rounds; per-step ms per round, median and
              spread (max - min) of each, and the median of the per-round differences
  conv_in   : ops.im2col3x3_nchw_cat + GEMM at K = 128 against ops.im2col3x3_nchw + GEMM at K = 64 on the UNet batch of
              a CFG step, over 200 launches between CUDA events (best of 3), with algorithmic bytes and FLOPs
  e2e_ms    : one StableDiffusionXLInpaintPipeline call with the 9-channel UNet (tensor image and mask,
              output_type="latent") after a warm-up call: preprocessing, two encodes, draws, the posterior kernel twice,
              the truncated denoise loop (graph replays), D2H of the latents; VAE decode not included
The card's name and power limit are read in the same process and reported with the numbers.
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def conv_in_cost(b: int, h: int, w: int, c_in: int, kpad: int, c_out: int = 320) -> dict:
    """Algorithmic bytes and FLOPs of conv_in as patch matrix + GEMM (fp16): the im2col kernel reads the c_in input
    channels once and writes the [b*h*w, kpad] matrix; the GEMM reads that matrix and the [c_out, kpad] weight and
    writes the [b*h*w, c_out] output, 2 * M * N * kpad FLOPs (the zero padding columns included, as the GEMM runs them)."""
    m = b * h * w
    im2col = 2 * (m * c_in + m * kpad)
    gemm = 2 * (m * kpad + c_out * kpad + c_out + m * c_out)
    return {"im2col_bytes": im2col, "gemm_bytes": gemm, "gemm_flop": 2 * m * c_out * kpad}


def measure(strength: float, K: int, res: int, rounds: int, replays: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE, SDXL_VAE
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    from tools.bench_img2img import card
    from tools.bench_inpaint import spread
    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint9 needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat = 1, res // 8
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLEncoder(SDXL_VAE))
    venc = AutoencoderKLEncoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 23, device=str(device)), device=device)
    unet4 = bench.build_native(SDXL_BASE, device)
    unet9 = bench.build_native(dataclasses.replace(SDXL_BASE, in_channels=9), device)
    pipe = StableDiffusionXLInpaintPipeline(unet9, vae_encoder=venc)
    eng9, eng4 = pipe.engine, DenoiseEngine(unet4)
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    g = torch.Generator("cpu").manual_seed(3)
    mask = torch.zeros((n, 1, lat, lat), dtype=torch.float16)
    mask[..., lat // 4:3 * lat // 4, lat // 4:3 * lat // 4] = 1
    masked = torch.randn((n, 4, lat, lat), generator=g).half()
    out = {"card": card(), "workload": f"SDXL-base UNet, CFG, n = {n}, {res}x{res}"}

    # ---- step graphs: capture both kinds, then replay them alternately
    args = (latents, pos, neg, pooled, npooled, tid, K)
    eng4.run(*args, guidance_scale=5.0, ip_scale=1.0)
    launches4 = eng4.last_launches_per_step
    eng9.run(*args, guidance_scale=5.0, ip_scale=1.0, begin_step=1, unet_cond=(mask, masked))
    out["launches_per_step"] = {"t2i": launches4, "inpaint9": eng9.last_launches_per_step}
    engines = {"t2i": eng4, "inpaint9": eng9}
    graphs = {kind: next(iter(e._graphs.values()))[0] for kind, e in engines.items()}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {"t2i": [], "inpaint9": []}
    for r in range(rounds):
        for kind in (("t2i", "inpaint9") if r % 2 == 0 else ("inpaint9", "t2i")):
            engines[kind]._restart(engines[kind]._loop, latents, 0)   # replays stay inside the K-step sigma table
            torch.cuda.synchronize()
            a.record()
            for _ in range(replays):
                graphs[kind].replay()
            b.record()
            torch.cuda.synchronize()
            times[kind].append(a.elapsed_time(b) / replays)
    diffs = [i - t for i, t in zip(times["inpaint9"], times["t2i"])]
    out["step_graph"] = {"replays_per_round": replays, "rounds": rounds,
                         "t2i_ms": spread(times["t2i"]), "inpaint9_ms": spread(times["inpaint9"]),
                         "inpaint9_minus_t2i_ms": spread(diffs)}

    # ---- conv_in alone: patch matrix + GEMM on the UNet batch of a CFG step
    B = 2 * n
    x0 = torch.randn((B, 4, lat, lat), generator=g).half().to(device)
    x1 = torch.cat([mask, masked], 1).repeat(2, 1, 1, 1).to(device)
    pair = {"t2i": lambda: ops.linear(ops.im2col3x3_nchw(x0, 64), unet4._w_in, unet4.conv_in.bias),
            "inpaint9": lambda: ops.linear(ops.im2col3x3_nchw_cat(x0, x1, 128), unet9._w_in, unet9.conv_in.bias)}
    reps = 200
    ct = {}
    for kind, fn in pair.items():
        ms = []
        for _ in range(3):
            fn()
            torch.cuda.synchronize()
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / reps)
        ct[kind] = min(ms)
    out["conv_in"] = {"note": f"{reps} launch pairs between CUDA events, best of 3; UNet batch {B}"}
    for kind, c_in, kpad in (("t2i", 4, 64), ("inpaint9", 9, 128)):
        cost = conv_in_cost(B, lat, lat, c_in, kpad)
        sec = ct[kind] * 1e-3
        out["conv_in"][kind] = {"us": ct[kind] * 1e3, **cost,
                                "tbps": (cost["im2col_bytes"] + cost["gemm_bytes"]) / sec / 1e12,
                                "gemm_tflops_over_pair_time": cost["gemm_flop"] / sec / 1e12}

    # ---- one 9-channel inpaint call end to end, no decode
    image = torch.rand((n, 3, res, res), generator=torch.Generator("cpu").manual_seed(5)) * 2 - 1
    pix_mask = torch.zeros((n, 1, res, res))
    pix_mask[..., res // 4:3 * res // 4, res // 4:3 * res // 4] = 1
    gen = torch.Generator(device).manual_seed(7)

    def call():
        return pipe(image=image, mask_image=pix_mask, strength=strength, num_inference_steps=K, height=res, width=res,
                    guidance_scale=5.0, generator=gen, prompt_embeds=pos, negative_prompt_embeds=neg,
                    pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=npooled,
                    output_type="latent").images.to("cpu")
    call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = call()
    torch.cuda.synchronize()
    out["e2e_ms"] = (time.perf_counter() - t0) * 1e3
    out["strength"], out["of_steps"] = strength, K
    out["steps_kept"] = K - eng9.scheduler.img2img_begin_index(K, strength)
    if not torch.isfinite(host.float()).all():
        raise RuntimeError("non-finite inpaint latents")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strength", type=float, default=0.6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    args = ap.parse_args()
    steps = max(2, args.steps)
    line = measure(args.strength, steps, args.res, args.rounds, min(args.replays, steps))
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_inpaint9.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
