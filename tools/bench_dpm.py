"""DPM-Solver++ 2M timing on one GPU: the DPM step graph against the Euler step graph, the two step kernels alone, and
one text-to-image call end to end with each scheduler.

    python tools/bench_dpm.py [--steps 20] [--res 1024] [--rounds 7] [--replays 10] [--karras 1]

Prints one JSON line.  Weights are random-init SDXL-base (UNet and IP processors), inputs are bench.py's synthetic
embeddings, n = 1, CFG 5.0.  No claim about image quality can rest on random weights; only time is measured.
  step_graph : the captured step graph of each scheduler (UNet forward + step kernel) replayed `replays` times
               between CUDA events, the two alternated over `rounds` rounds; per-step ms per round, median and spread
               (max - min) of each, and of the per-round differences
  step_kernel: ops.dpm_solver_step and ops.euler_step (each with its step-counter increment) over 200 launches
               between CUDA events, best of 3; the DPM kernel's algorithmic bytes (dpm_step_bytes) and their rate
               against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM
  e2e_ms     : one StableDiffusionXLCustomPipeline call per scheduler (output_type="latent", `steps` steps) after a
               warm-up call: prompt embeddings given, latents drawn, the graph-replayed loop, D2H of the latents
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


def dpm_step_bytes(n: int, C: int, h: int, w: int, cfg: bool) -> int:
    """Algorithmic HBM bytes of one second-order ih_dpm_solver_step (fp16): reads the noise prediction (2n images with
    CFG), the latents and the previous x0; writes the latents, x0 and the next model input (2n images with CFG).  The
    step counter, loop_begin and the 32-byte coefficient row are not counted."""
    b = 2 * n if cfg else n
    img = C * h * w
    return 2 * ((b + 2 * n) * img + (2 * n + b) * img)


def euler_step_bytes(n: int, C: int, h: int, w: int, cfg: bool) -> int:
    """The same count for the Euler step kernel (no previous x0 read or x0 written)."""
    return dpm_step_bytes(n, C, h, w, cfg) - 2 * 2 * n * C * h * w


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs)}


def measure(K: int, res: int, rounds: int, replays: int, karras: bool) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    from tools.bench_img2img import card
    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat = 1, res // 8
    unet = bench.build_native(SDXL_BASE, device)
    scheds = {"euler": EulerDiscreteScheduler(), "dpm": DPMSolverMultistepScheduler(use_karras_sigmas=karras)}
    engines = {k: DenoiseEngine(unet, scheduler=s) for k, s in scheds.items()}
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    out = {"card": card(), "workload": f"SDXL-base UNet, CFG 5.0, n = {n}, {res}x{res}",
           "dpm": scheds["dpm"].kind}

    # ---- step graphs: capture both kinds, then replay them alternately from the same start state
    args = (latents, pos, neg, pooled, npooled, tid, K)
    for eng in engines.values():
        eng.run(*args, guidance_scale=5.0, ip_scale=1.0)
    graphs = {k: next(iter(eng._graphs.values()))[0] for k, eng in engines.items()}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {"euler": [], "dpm": []}
    for r in range(rounds):
        for kind in (("euler", "dpm") if r % 2 == 0 else ("dpm", "euler")):
            eng = engines[kind]
            st = eng._loop.st
            eng.unet.prepare_conditioning(st["ehs"], st["text_embeds"], st["time_ids"])
            eng._restart(eng._loop, latents, 0)                 # replays stay inside the K-step tables
            torch.cuda.synchronize()
            a.record()
            for _ in range(replays):
                graphs[kind].replay()
            b.record()
            torch.cuda.synchronize()
            times[kind].append(a.elapsed_time(b) / replays)
    diffs = [d - e for d, e in zip(times["dpm"], times["euler"])]
    out["step_graph"] = {"replays_per_round": replays, "rounds": rounds, "euler_ms": spread(times["euler"]),
                         "dpm_ms": spread(times["dpm"]), "dpm_minus_euler_ms": spread(diffs)}

    # ---- the two step kernels alone (each launch: step kernel + step-counter increment)
    g = torch.Generator("cpu").manual_seed(3)
    sig = engines["euler"].tables(K)[1]
    coeffs = engines["dpm"].coeffs(K)
    step = torch.zeros((1,), dtype=torch.int32, device=device)
    loop_begin = torch.zeros((1,), dtype=torch.int32, device=device)
    pred = torch.randn((2 * n, 4, lat, lat), generator=g).half().to(device)
    x = torch.randn((n, 4, lat, lat), generator=g).half().to(device)
    x0 = torch.randn((n, 4, lat, lat), generator=g).half().to(device)
    mi = torch.empty((2 * n, 4, lat, lat), dtype=torch.float16, device=device)
    kern = {"euler": lambda: ops.euler_step(pred, x, mi, sig, step, 5.0),
            "dpm": lambda: ops.dpm_solver_step(pred, x, mi, x0, coeffs, step, loop_begin, 5.0)}
    reps = 200
    kt = {}
    for kind, fn in kern.items():
        ms = []
        for _ in range(3):
            step.zero_()
            fn()
            torch.cuda.synchronize()
            a.record()
            for k in range(reps):
                if k % (K - 1) == 0:
                    step.fill_(1)                               # second-order steps only (index 1 .. K-2) for DPM
                fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / reps)
        kt[kind] = min(ms)
    by = dpm_step_bytes(n, 4, lat, lat, True)
    out["step_kernel"] = {
        "note": f"{reps} launches between CUDA events, best of 3; a step.fill_() every {K - 1} launches is inside the "
                "window for both kinds",
        "euler_us": kt["euler"] * 1e3, "dpm_us": kt["dpm"] * 1e3,
        "dpm_bytes_algorithmic": by, "euler_bytes_algorithmic": euler_step_bytes(n, 4, lat, lat, True),
        "dpm_tbps": by / (kt["dpm"] * 1e-3) / 1e12,
        "dpm_frac_of_hbm_datasheet": by / (kt["dpm"] * 1e-3) / 1e12 / HBM_TBPS_DATASHEET}

    # ---- one text-to-image call per scheduler, end to end, no decode
    out["e2e_ms"] = {}
    for kind, s in scheds.items():
        pipe = StableDiffusionXLCustomPipeline(unet, scheduler=s)

        def call():
            return pipe(num_inference_steps=K, height=res, width=res, guidance_scale=5.0,
                        generator=torch.Generator("cpu").manual_seed(7), prompt_embeds=pos, negative_prompt_embeds=neg,
                        pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=npooled,
                        output_type="latent").images.to("cpu")
        call()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = call()
        torch.cuda.synchronize()
        out["e2e_ms"][kind] = (time.perf_counter() - t0) * 1e3
        if not torch.isfinite(host.float()).all():
            raise RuntimeError(f"non-finite {kind} latents")
    out["steps"] = K
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    ap.add_argument("--karras", type=int, default=1)
    args = ap.parse_args()
    steps = max(3, args.steps)
    line = measure(steps, args.res, args.rounds, min(args.replays, steps), bool(args.karras))
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
