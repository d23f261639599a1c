"""UniPC timing on one GPU: the UniPC step graph against the DPM-Solver++ and Euler step graphs, the UniPC step kernel
alone, and text-to-image calls end to end with UniPC at 10 steps against DPM++ 2M Karras at 20 and 25.

    python tools/bench_unipc.py [--res 1024] [--rounds 7] [--replays 10]

Prints one JSON line.  Weights are random-init SDXL-base (UNet and IP processors), inputs are bench.py's synthetic
embeddings, n = 1, CFG 5.0.  No claim about image quality can rest on random weights; only time is measured.
  step_graph : the captured step graph of each scheduler (UNet forward + step kernel) replayed `replays` times
               between CUDA events, the three alternated over `rounds` rounds (order rotated); per-step ms per round,
               median and spread (max - min) of each
  step_kernel: the UniPC, DPM-Solver++ and Euler step kernels (ops.dpm_solver_step with and without unipc=, and
               ops.euler_step), each with its step-counter increment, over 200 launches between CUDA events with no
               other work in the window, alternated, best of 3; UniPC at steps with corrector and predictor of order 2,
               DPM at second-order steps.  Their algorithmic bytes (unipc_step_bytes, bench_dpm's dpm_step_bytes and
               euler_step_bytes) and rates, and UniPC's rate against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM
  e2e_ms     : one StableDiffusionXLCustomPipeline call per configuration (output_type="latent") after a warm-up call:
               prompt embeddings given, latents drawn, the graph-replayed loop, D2H of the latents
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

from tools.bench_dpm import HBM_TBPS_DATASHEET, spread  # noqa: E402

E2E = (("unipc", 10), ("dpmpp_2m_karras", 20), ("dpmpp_2m_karras", 25))


def unipc_step_bytes(n: int, C: int, h: int, w: int, cfg: bool) -> int:
    """Algorithmic HBM bytes of one ih_dpm_solver_step with IH_SOLVER_UNIPC_BH2 (fp16) at orders 2 / 2: reads the noise
    prediction (2n images with CFG), the latents, last_sample, prev_x0 and prev_x0_2; writes the latents, last_sample,
    prev_x0, prev_x0_2 and the next model input (2n images with CFG).  The step counter, loop_begin and the 64-byte
    coefficient row are not counted."""
    b = 2 * n if cfg else n
    img = C * h * w
    return 2 * ((b + 4 * n) * img + (4 * n + b) * img)


def measure(res: int, rounds: int, replays: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler, UniPCMultistepScheduler
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    from tools.bench_img2img import card
    if not torch.cuda.is_available():
        raise SystemExit("bench_unipc needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat, K = 1, res // 8, 10
    unet = bench.build_native(SDXL_BASE, device)
    make = {"euler": EulerDiscreteScheduler,
            "dpmpp_2m_karras": lambda: DPMSolverMultistepScheduler(use_karras_sigmas=True),
            "unipc": UniPCMultistepScheduler}
    engines = {k: DenoiseEngine(unet, scheduler=f()) for k, f in make.items()}
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    out = {"card": card(), "workload": f"SDXL-base UNet, CFG 5.0, n = {n}, {res}x{res}"}

    # ---- step graphs: capture each kind, then replay them in rotated order from the same start state
    args = (latents, pos, neg, pooled, npooled, tid, K)
    for eng in engines.values():
        eng.run(*args, guidance_scale=5.0, ip_scale=1.0)
    graphs = {k: next(iter(eng._graphs.values()))[0] for k, eng in engines.items()}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kinds = list(engines)
    times = {k: [] for k in kinds}
    for r in range(rounds):
        for kind in kinds[r % 3:] + kinds[:r % 3]:
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
    out["step_graph"] = {"replays_per_round": replays, "rounds": rounds, "steps": K,
                         **{f"{k}_ms": spread(v) for k, v in times.items()}}

    # ---- the step kernels alone (each launch: step kernel + step-counter increment).  The tables are reps + 4 steps
    # long, so the counter walks steps 2 .. reps + 1 (UniPC: corrector and predictor of order 2; DPM: second order)
    # without a reset inside the timed window.
    from tools.bench_dpm import dpm_step_bytes, euler_step_bytes
    reps = 200
    Tk = reps + 4
    g = torch.Generator("cpu").manual_seed(3)
    tables = {}
    for kind, sched in (("unipc", UniPCMultistepScheduler()), ("dpm", DPMSolverMultistepScheduler()),
                        ("euler", EulerDiscreteScheduler())):
        sched.set_timesteps(Tk)
        tables[kind] = torch.from_numpy(sched.coeffs if kind != "euler" else sched.sigmas).to(device)
    step = torch.zeros((1,), dtype=torch.int32, device=device)
    loop_begin = torch.zeros((1,), dtype=torch.int32, device=device)
    pred = torch.randn((2 * n, 4, lat, lat), generator=g).half().to(device)
    x, ls, x0, x0_2 = (torch.randn((n, 4, lat, lat), generator=g).half().to(device) for _ in range(4))
    mi = torch.empty((2 * n, 4, lat, lat), dtype=torch.float16, device=device)
    kern = {"unipc": lambda: ops.dpm_solver_step(pred, x, mi, x0, tables["unipc"], step, loop_begin, 5.0,
                                                 unipc=(ls, x0_2)),
            "dpm": lambda: ops.dpm_solver_step(pred, x, mi, x0, tables["dpm"], step, loop_begin, 5.0),
            "euler": lambda: ops.euler_step(pred, x, mi, tables["euler"], step, 5.0)}
    kt = {k: [] for k in kern}
    for r in range(3):                                          # kinds alternated, best of 3 per kind
        for kind in list(kern)[r:] + list(kern)[:r]:
            step.fill_(1)
            kern[kind]()                                        # step 1 (warm), leaves the counter at 2
            torch.cuda.synchronize()
            a.record()
            for _ in range(reps):
                kern[kind]()
            b.record()
            torch.cuda.synchronize()
            kt[kind].append(a.elapsed_time(b) / reps)
    best = {k: min(v) for k, v in kt.items()}
    by = {"unipc": unipc_step_bytes(n, 4, lat, lat, True), "dpm": dpm_step_bytes(n, 4, lat, lat, True),
          "euler": euler_step_bytes(n, 4, lat, lat, True)}
    out["step_kernel"] = {
        "note": f"{reps} launches between CUDA events per kind, no other work in the window, kinds alternated, best "
                "of 3",
        **{f"{k}_us": best[k] * 1e3 for k in kern},
        **{f"{k}_bytes_algorithmic": by[k] for k in kern},
        **{f"{k}_tbps": by[k] / (best[k] * 1e-3) / 1e12 for k in kern},
        "unipc_frac_of_hbm_datasheet": by["unipc"] / (best["unipc"] * 1e-3) / 1e12 / HBM_TBPS_DATASHEET}

    # ---- text-to-image calls end to end, no decode
    out["e2e_ms"] = {}
    for kind, steps in E2E:
        pipe = StableDiffusionXLCustomPipeline(unet, scheduler=make[kind]())

        def call():
            return pipe(num_inference_steps=steps, height=res, width=res, guidance_scale=5.0,
                        generator=torch.Generator("cpu").manual_seed(7), prompt_embeds=pos, negative_prompt_embeds=neg,
                        pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=npooled,
                        output_type="latent").images.to("cpu")
        call()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = call()
        torch.cuda.synchronize()
        out["e2e_ms"][f"{kind}_{steps}"] = (time.perf_counter() - t0) * 1e3
        if not torch.isfinite(host.float()).all():
            raise RuntimeError(f"non-finite {kind} latents")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    args = ap.parse_args()
    print(json.dumps(measure(args.res, args.rounds, min(args.replays, 10))), flush=True)


if __name__ == "__main__":
    main()
