"""Inpainting timing on one GPU: the inpaint step graph against the text-to-image step graph, the fused Euler + blend
kernel against the plain Euler kernel, and one inpaint call end to end.

    python tools/bench_inpaint.py [--strength 0.6] [--steps 20] [--res 1024] [--rounds 7] [--replays 10]

Prints one JSON line and writes it to tools_out/bench_inpaint.json.  Weights are random-init SDXL-base (UNet, IP
processors, VAE encoder), inputs are bench.py's synthetic embeddings, the mask regenerates the middle half of the image.
  step_graph : the captured step graph of each kind (UNet forward + Euler kernel, CFG, n = 1) replayed `replays` times
               between CUDA events, the two kinds alternated over `rounds` rounds; per-step ms per round, median and
               spread (max - min) of each, and the median of the per-round differences
  step_kernel: ops.euler_inpaint_step and ops.euler_step (each with its step-counter increment) over 200 launches
               between CUDA events; the inpaint kernel's algorithmic bytes (inpaint_step_bytes) and their rate against
               the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM
  e2e_ms     : one StableDiffusionXLInpaintPipeline call (tensor image and mask, output_type="latent") after a warm-up
               call: preprocessing, encode, eps / noise draws, the posterior kernel twice, the truncated denoise loop
               (graph replays), D2H of the latents; VAE decode not included
The card's name and power limit are read in the same process and reported with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS_DATASHEET = 3.35          # H100 SXM HBM3, NVIDIA data sheet


def inpaint_step_bytes(n: int, C: int, h: int, w: int, cfg: bool) -> int:
    """Algorithmic HBM bytes of one ih_euler_inpaint_step (fp16): reads the noise prediction (2n images with CFG),
    the latents, the image latents, the blend noise and the one-channel mask; writes the latents and the next model
    input (2n images with CFG).  The step counter, sigmas and blend_end are a few bytes and not counted."""
    b = 2 * n if cfg else n
    img = C * h * w
    reads = b * img + n * img + 2 * n * img + n * h * w
    writes = n * img + b * img
    return 2 * (reads + writes)


def euler_step_bytes(n: int, C: int, h: int, w: int, cfg: bool) -> int:
    """The same count for the text-to-image step kernel (no image latents, blend noise or mask)."""
    return inpaint_step_bytes(n, C, h, w, cfg) - 2 * (2 * n * C * h * w + n * h * w)


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs)}


def measure(strength: float, K: int, res: int, rounds: int, replays: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE, SDXL_VAE
    from imagharmony_b200.vae import AutoencoderKLEncoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLInpaintPipeline
    from tools.bench_img2img import card
    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat = 1, res // 8
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLEncoder(SDXL_VAE))
    venc = AutoencoderKLEncoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 23, device=str(device)), device=device)
    pipe = StableDiffusionXLInpaintPipeline(bench.build_native(SDXL_BASE, device), vae_encoder=venc)
    eng = pipe.engine
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    g = torch.Generator("cpu").manual_seed(3)
    image_latents = torch.randn((n, 4, lat, lat), generator=g).half().to(device)
    noise = torch.randn((n, 4, lat, lat), generator=g).half().to(device)
    mask = torch.zeros((n, 1, lat, lat), dtype=torch.float16)
    mask[..., lat // 4:3 * lat // 4, lat // 4:3 * lat // 4] = 1
    mask = mask.to(device)
    out = {"card": card(), "workload": f"SDXL-base UNet, CFG, n = {n}, {res}x{res}"}

    # ---- step graphs: capture both kinds, then replay them alternately
    args = (latents, pos, neg, pooled, npooled, tid, K)
    eng.run(*args, guidance_scale=5.0, ip_scale=1.0)
    eng.run(*args, guidance_scale=5.0, ip_scale=1.0, inpaint=(image_latents, noise, mask))
    graphs = {kind: next(g for key, (g, _) in eng._graphs.items() if key.ib == (kind == "inpaint"))
              for kind in ("t2i", "inpaint")}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {"t2i": [], "inpaint": []}
    for r in range(rounds):
        for kind in (("t2i", "inpaint") if r % 2 == 0 else ("inpaint", "t2i")):
            eng._restart(eng._loop, latents, 0)                # replays stay inside the K-step sigma table
            torch.cuda.synchronize()
            a.record()
            for _ in range(replays):
                graphs[kind].replay()
            b.record()
            torch.cuda.synchronize()
            times[kind].append(a.elapsed_time(b) / replays)
    diffs = [i - t for i, t in zip(times["inpaint"], times["t2i"])]
    out["step_graph"] = {"replays_per_round": replays, "rounds": rounds,
                         "t2i_ms": spread(times["t2i"]), "inpaint_ms": spread(times["inpaint"]),
                         "inpaint_minus_t2i_ms": spread(diffs)}

    # ---- the two step kernels alone (each launch: step kernel + step-counter increment)
    sig = eng.tables(K)[1]
    step = torch.zeros((1,), dtype=torch.int32, device=device)
    blend_end = torch.full((1,), K, dtype=torch.int32, device=device)
    pred = torch.randn((2 * n, 4, lat, lat), generator=g).half().to(device)
    x = latents.to(device)
    mi = torch.empty((2 * n, 4, lat, lat), dtype=torch.float16, device=device)
    kern = {"t2i": lambda: ops.euler_step(pred, x, mi, sig, step, 5.0),
            "inpaint": lambda: ops.euler_inpaint_step(pred, x, mi, sig, step, 5.0, image_latents, noise, mask, blend_end)}
    reps = 200
    kt = {}
    for kind, fn in kern.items():
        ms = []
        for _ in range(3):
            step.zero_()
            fn()
            torch.cuda.synchronize()
            step.zero_()
            a.record()
            for k in range(reps):
                if k % (K - 1) == 0:
                    step.zero_()
                fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / reps)
        kt[kind] = min(ms)
    by = inpaint_step_bytes(n, 4, lat, lat, True)
    out["step_kernel"] = {
        "note": f"{reps} launches between CUDA events, best of 3; a step.zero_() every {K - 1} launches is inside the "
                "window for both kinds",
        "t2i_us": kt["t2i"] * 1e3, "inpaint_us": kt["inpaint"] * 1e3,
        "inpaint_bytes_algorithmic": by, "t2i_bytes_algorithmic": euler_step_bytes(n, 4, lat, lat, True),
        "inpaint_tbps": by / (kt["inpaint"] * 1e-3) / 1e12,
        "inpaint_frac_of_hbm_datasheet": by / (kt["inpaint"] * 1e-3) / 1e12 / HBM_TBPS_DATASHEET}

    # ---- one inpaint call end to end, no decode
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
    out["steps_kept"] = K - eng.scheduler.img2img_begin_index(K, strength)
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
    with open(os.path.join(ROOT, "tools_out", "bench_inpaint.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
