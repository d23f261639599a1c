"""Multi-ControlNet timing on one GPU: step graphs with 0, 1 and 2 ControlNets, the fused injection kernel for K = 1, 2,
3 nets against its algorithmic bytes, one two-net pipeline call end to end, and the peak device memory of a two-net
call with staggered guidance windows.

    python tools/bench_multi_controlnet.py [--steps 20] [--res 1024] [--rounds 7] [--replays 10]

Prints one JSON line and writes it to tools_out/bench_multi_controlnet.json.  Weights are random-init SDXL-base UNet
(IP processors) and two random SDXL ControlNets; inputs are bench.py's synthetic embeddings and random control images.
  step_graph : the captured step graph of each arm (CFG, n = 1): text-to-image (0 nets), one ControlNet, two
               ControlNets; each replayed `replays` times between CUDA events, the arms alternated over `rounds`
               rounds; per-step ms per round, median and spread (max - min), launches per step
  injection  : ops.controlnet_add_residuals_multi on the 10 SDXL skip shapes of a CFG step for K = 1, 2, 3 nets, 200
               launches between CUDA events (best of 3), against its algorithmic bytes ((2 + K) x the touched skip
               bytes: the skips read and written, K residuals read) and the 3.35 TB/s HBM3 data-sheet figure of the
               H100 SXM
  e2e_ms     : one two-net StableDiffusionXLControlNetPipeline call (tensor control images, output_type="latent")
               after a warm-up call
  peak_mem   : torch.cuda.max_memory_allocated over a two-net call with windows [0, 0.5] and [0.25, 1] (3 graphs
               captured), on a fresh pipeline
The card's name, power limit and maximum SM clock are read in the same process and reported with the numbers.
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

from tools.bench_controlnet import HBM3_TBPS, injection_bytes, skip_shapes  # noqa: E402


def multi_injection_bytes(shapes, batch: int, rows_batch: int, nets: int) -> dict:
    """Algorithmic fp16 bytes of ih_controlnet_add_residuals_multi_f16 with `nets` nets: the touched skip rows are read
    and written once and each net's residuals read once, (2 + nets) x the touched skip bytes."""
    one = injection_bytes(shapes, batch, rows_batch)
    return {"skip_bytes": one["skip_bytes"], "touched_skip_bytes": one["touched_skip_bytes"],
            "algorithmic_bytes": (2 + nets) * one["touched_skip_bytes"]}


def card() -> dict:
    """Name, power limit and maximum SM clock of GPU 0, from nvidia-smi in this process."""
    import subprocess
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:      # report what failed rather than a made-up card
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi_error": repr(e)}


def measure(K: int, res: int, rounds: int, replays: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetCall, ControlNetModel
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    from tools.bench_inpaint import spread
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_controlnet needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat = 1, res // 8
    unet = bench.build_native(SDXL_BASE, device)
    with torch.device("meta"):
        shapes = shapes_of(ControlNetModel(SDXL_CONTROLNET))
    nets = [ControlNetModel.from_state_dict(SDXL_CONTROLNET, random_state_dict(shapes, s, device=str(device)),
                                            device=device) for s in (29, 31)]
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    images = [torch.rand((n, 3, res, res), generator=torch.Generator("cpu").manual_seed(5 + j)) for j in range(2)]
    out = {"card": card(), "workload": f"SDXL-base UNet + 2 SDXL ControlNets, CFG, n = {n}, {res}x{res}"}

    # ---- step graphs with 0, 1, 2 nets: one engine per arm (each holds one graph), replayed alternately
    args = (latents, pos, neg, pooled, npooled, tid, K)
    calls = [ControlNetCall(m, im.half(), 1.0, False) for m, im in zip(nets, images)]
    engines = {"nets0": DenoiseEngine(unet), "nets1": DenoiseEngine(unet), "nets2": DenoiseEngine(unet)}
    engines["nets0"].run(*args, guidance_scale=5.0, ip_scale=1.0)
    engines["nets1"].run(*args, guidance_scale=5.0, ip_scale=1.0, controlnet=calls[0])
    engines["nets2"].run(*args, guidance_scale=5.0, ip_scale=1.0, controlnet=calls)
    out["launches_per_step"] = {}
    graphs = {}
    for kind, e in engines.items():
        assert len(e._graphs) == 1, (kind, list(e._graphs))
        graphs[kind] = next(iter(e._graphs.values()))[0]
        out["launches_per_step"][kind] = e.last_launches_per_step
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {k: [] for k in engines}
    order = list(engines)
    for r in range(rounds):
        for kind in order[r % 3:] + order[:r % 3]:
            engines[kind]._restart(engines[kind]._loop, latents, 0)   # replays stay inside the K-step sigma table
            torch.cuda.synchronize()
            a.record()
            for _ in range(replays):
                graphs[kind].replay()
            b.record()
            torch.cuda.synchronize()
            times[kind].append(a.elapsed_time(b) / replays)
    out["step_graph"] = {"replays_per_round": replays, "rounds": rounds,
                         **{f"{k}_ms": spread(v) for k, v in times.items()},
                         **{f"{k}_minus_nets0_ms": spread([x - t for x, t in zip(times[k], times["nets0"])])
                            for k in ("nets1", "nets2")}}
    del engines, graphs
    torch.cuda.empty_cache()

    # ---- the fused injection kernel alone on the SDXL skip shapes of a CFG step, K = 1, 2, 3
    g = torch.Generator("cpu").manual_seed(3)
    sh = skip_shapes(SDXL_BASE.block_out_channels, SDXL_BASE.layers_per_block, lat)
    B = 2 * n
    skips = [torch.randn((B, h, w, c), generator=g).half().to(device) for h, w, c in sh]
    res_t = [[torch.randn((B * h * w, c), generator=g).half().to(device) * 1e-3 for h, w, c in sh] for _ in range(3)]
    scale = torch.full((10,), 0.5, dtype=torch.float32, device=device)
    out["injection"] = {}
    reps = 200
    for k in (1, 2, 3):
        ms = []
        for _ in range(3):
            ops.controlnet_add_residuals_multi(skips, res_t[:k], [scale] * k, [0] * 10)
            torch.cuda.synchronize()
            a.record()
            for _ in range(reps):
                ops.controlnet_add_residuals_multi(skips, res_t[:k], [scale] * k, [0] * 10)
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / reps)
        cost = multi_injection_bytes(sh, B, B, k)
        tbps = cost["algorithmic_bytes"] / (min(ms) * 1e-3) / 1e12
        out["injection"][f"K{k}"] = {"us": min(ms) * 1e3, **cost, "tbps": tbps,
                                     "frac_of_datasheet_hbm": tbps / HBM3_TBPS}
    out["injection"]["note"] = f"{reps} launches between CUDA events, best of 3; UNet batch {B}"
    del skips, res_t

    # ---- one two-net pipeline call end to end, no decode
    pipe = StableDiffusionXLControlNetPipeline(unet, nets)
    gen = torch.Generator(device).manual_seed(7)

    def call(p, **kw):
        return p(image=images, num_inference_steps=K, guidance_scale=5.0, generator=gen, prompt_embeds=pos,
                 negative_prompt_embeds=neg, pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=npooled,
                 output_type="latent", **kw).images.to("cpu")
    call(pipe)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = call(pipe)
    torch.cuda.synchronize()
    out["e2e_ms"] = (time.perf_counter() - t0) * 1e3
    out["of_steps"] = K
    if not torch.isfinite(host.float()).all():
        raise RuntimeError("non-finite Multi-ControlNet latents")
    del pipe
    torch.cuda.empty_cache()

    # ---- peak device memory of a two-net call with staggered windows (3 graphs), on a fresh pipeline
    pipe = StableDiffusionXLControlNetPipeline(unet, nets)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    call(pipe, control_guidance_start=[0.0, 0.25], control_guidance_end=[0.5, 1.0])
    torch.cuda.synchronize()
    out["peak_mem"] = {"peak_gib": torch.cuda.max_memory_allocated() / 2**30,
                       "before_call_gib": before / 2**30, "graphs_captured": pipe.engine.graphs_captured}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    args = ap.parse_args()
    steps = max(4, args.steps)
    line = measure(steps, args.res, args.rounds, min(args.replays, steps))
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_multi_controlnet.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
