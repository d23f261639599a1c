"""ControlNet timing on one GPU: the ControlNet step graph (guess mode as a third arm) against the text-to-image step
graph, the residual-injection kernel against its algorithmic bytes, the once-per-call conditioning embedding, and one
ControlNet pipeline call end to end.

    python tools/bench_controlnet.py [--steps 20] [--res 1024] [--rounds 7] [--replays 10]

Prints one JSON line and writes it to tools_out/bench_controlnet.json.  Weights are random-init SDXL-base UNet (IP
processors) and SDXL ControlNet; inputs are bench.py's synthetic embeddings and a random control image.
  step_graph : the captured step graph of each arm (CFG, n = 1): text-to-image (UNet + Euler kernel), ControlNet
               (ControlNet on the CFG batch + UNet with the residuals injected + Euler kernel), guess mode (the
               ControlNet on the conditional half); each replayed `replays` times between CUDA events, the arms
               alternated over `rounds` rounds; per-step ms per round, median and spread (max - min) of each, and the
               median of the per-round differences against text-to-image
  injection  : ops.controlnet_add_residuals on the 10 SDXL skip shapes of a CFG step, 200 launches between CUDA events
               (best of 3), against its algorithmic bytes (the skips read and written, the residuals read) and the
               3.35 TB/s HBM3 data-sheet figure of the H100 SXM
  embedding  : ControlNetModel.embed_condition of one control image (once per call), with its algorithmic FLOPs
  e2e_ms     : one StableDiffusionXLControlNetPipeline call (tensor control image, output_type="latent") after a warm-up
               call: preprocessing, embedding, prompt conditioning, the denoise loop (graph replays), D2H of the latents
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

HBM3_TBPS = 3.35          # NVIDIA H100 SXM data sheet (700 W card)


def skip_shapes(block_out_channels, layers_per_block: int, lat: int):
    """(h, w, C) of the ControlNet's 10 residuals, which are the UNet's 9 skips then the mid-block output: conv_in, then
    per level its `layers_per_block` resnet/attention outputs and (all but the last level) its downsampler."""
    shapes = [(lat, lat, block_out_channels[0])]
    side = lat
    for i, c in enumerate(block_out_channels):
        shapes += [(side, side, c)] * layers_per_block
        if i < len(block_out_channels) - 1:
            side //= 2
            shapes.append((side, side, c))
    return shapes + [(side, side, block_out_channels[-1])]


def injection_bytes(shapes, batch: int, rows_batch: int) -> dict:
    """Algorithmic fp16 bytes of ih_controlnet_add_residuals_f16: the skip tensors of a `batch`-image UNet batch, of
    which `rows_batch` images get residuals (the whole batch, or the conditional half in guess mode); those skip rows
    are read and written and the residuals read once."""
    skip = sum(2 * batch * h * w * c for h, w, c in shapes)
    touched = sum(2 * rows_batch * h * w * c for h, w, c in shapes)
    return {"skip_bytes": skip, "touched_skip_bytes": touched, "algorithmic_bytes": 3 * touched}


def embedding_flop(res_h: int, res_w: int, widths, out_channels: int, in_channels: int = 3) -> int:
    """FLOPs of the conditioning embedding of one image: conv_in, the stride-1 / stride-2 conv pairs, conv_out; every
    conv 3x3, pad 1, 2 * Ho * Wo * Cout * Cin * 9."""
    flop, h, w = 2 * res_h * res_w * widths[0] * in_channels * 9, res_h, res_w
    for c, c2 in zip(widths[:-1], widths[1:]):
        flop += 2 * h * w * c * c * 9
        h, w = (h + 1) // 2, (w + 1) // 2
        flop += 2 * h * w * c2 * c * 9
    return flop + 2 * h * w * out_channels * widths[-1] * 9


def measure(K: int, res: int, rounds: int, replays: int) -> dict:
    import bench
    from imagharmony_b200 import ops
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetCall, ControlNetModel
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    from tools.bench_img2img import card
    from tools.bench_inpaint import spread
    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet needs a GPU")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    n, lat = 1, res // 8
    unet = bench.build_native(SDXL_BASE, device)
    with torch.device("meta"):
        shapes = shapes_of(ControlNetModel(SDXL_CONTROLNET))
    cn = ControlNetModel.from_state_dict(SDXL_CONTROLNET, random_state_dict(shapes, 29, device=str(device)),
                                         device=device)
    latents, pos, neg, pooled, npooled, tid = bench.synth_inputs(SDXL_BASE, n, lat, K, 0)
    image = torch.rand((n, 3, res, res), generator=torch.Generator("cpu").manual_seed(5))
    out = {"card": card(), "workload": f"SDXL-base UNet + SDXL ControlNet, CFG, n = {n}, {res}x{res}"}

    # ---- step graphs: one engine per arm (each holds one graph), replayed alternately
    args = (latents, pos, neg, pooled, npooled, tid, K)
    engines = {"t2i": DenoiseEngine(unet), "controlnet": DenoiseEngine(unet), "guess": DenoiseEngine(unet)}
    engines["t2i"].run(*args, guidance_scale=5.0, ip_scale=1.0)
    for kind, guess in (("controlnet", False), ("guess", True)):
        engines[kind].run(*args, guidance_scale=5.0, ip_scale=1.0,
                          controlnet=ControlNetCall(cn, image.half(), 1.0, guess))
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
                         **{f"{k}_minus_t2i_ms": spread([x - t for x, t in zip(times[k], times["t2i"])])
                            for k in ("controlnet", "guess")}}

    # ---- the injection kernel alone on the SDXL skip shapes of a CFG step
    g = torch.Generator("cpu").manual_seed(3)
    sh = skip_shapes(SDXL_BASE.block_out_channels, SDXL_BASE.layers_per_block, lat)
    B = 2 * n
    skips = [torch.randn((B, h, w, c), generator=g).half().to(device) for h, w, c in sh]
    res_t = [torch.randn((B * h * w, c), generator=g).half().to(device) * 1e-3 for h, w, c in sh]
    scale = torch.full((10,), 0.5, dtype=torch.float32, device=device)
    reps, ms = 200, []
    for _ in range(3):
        ops.controlnet_add_residuals(skips, res_t, scale, [0] * 10)
        torch.cuda.synchronize()
        a.record()
        for _ in range(reps):
            ops.controlnet_add_residuals(skips, res_t, scale, [0] * 10)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / reps)
    cost = injection_bytes(sh, B, B)
    tbps = cost["algorithmic_bytes"] / (min(ms) * 1e-3) / 1e12
    out["injection"] = {"us": min(ms) * 1e3, **cost, "tbps": tbps, "frac_of_datasheet_hbm": tbps / HBM3_TBPS,
                        "note": f"{reps} launches between CUDA events, best of 3; UNet batch {B}"}

    # ---- the conditioning embedding of one control image (once per call)
    img16 = image.half().to(device)
    ms = []
    for _ in range(3):
        cn.embed_condition(img16)
        torch.cuda.synchronize()
        a.record()
        for _ in range(10):
            cn.embed_condition(img16)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / 10)
    flop = embedding_flop(res, res, SDXL_CONTROLNET.conditioning_embedding_out_channels, SDXL_BASE.block_out_channels[0])
    out["embedding"] = {"ms": min(ms), "flop": flop, "tflops": flop / (min(ms) * 1e-3) / 1e12,
                        "note": "10 calls between CUDA events, best of 3; one image"}

    # ---- one ControlNet pipeline call end to end, no decode
    pipe = StableDiffusionXLControlNetPipeline(unet, cn)
    gen = torch.Generator(device).manual_seed(7)

    def call():
        return pipe(image=image, num_inference_steps=K, guidance_scale=5.0, generator=gen, prompt_embeds=pos,
                    negative_prompt_embeds=neg, pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=npooled,
                    output_type="latent").images.to("cpu")
    call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = call()
    torch.cuda.synchronize()
    out["e2e_ms"] = (time.perf_counter() - t0) * 1e3
    out["of_steps"] = K
    if not torch.isfinite(host.float()).all():
        raise RuntimeError("non-finite ControlNet latents")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    args = ap.parse_args()
    steps = max(2, args.steps)
    line = measure(steps, args.res, args.rounds, min(args.replays, steps))
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tools_out", "bench_controlnet.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
