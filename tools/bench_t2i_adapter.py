"""The SDXL T2I-Adapter on one GPU: its once-per-call forward, its cost per denoise step, and a whole call against
one with a ControlNet.

    python tools/bench_t2i_adapter.py [--warmup 2] [--iters 5] [--rounds 6] [--replays 20] [--steps 30] [--out tools_out]

* The adapter forward (random-init full_adapter_xl weights, SDXL widths) at every SDXL bucket for batches 1 and 4:
  median of `iters` CUDA-event timings after `warmup` calls, with the FLOPs and bytes counted from the shapes here
  (adapter_cost) and which bound (H100 SXM data-sheet compute or HBM bandwidth) is the larger.
* The 1024^2 CFG step (SDXL-base UNet, batch 1) with and without an active adapter: the two step graphs the engine
  captured, replayed `replays` times per timing, in `rounds` alternated rounds (the order flips every round); median
  per-step time of each and the spread (max - min over rounds), plus the injection's algorithmic bytes
  (injection_bytes).
* One `steps`-step 1024^2 call (latent output) with the adapter against the same call with one SDXL ControlNet.

The card's name, power limit and max SM clock are read in the same process and printed with the numbers.  One JSON
line per measurement; all lines also go to <out>/bench_t2i_adapter.json.
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
    """(FLOPs, bytes) of a k x k conv over P output pixels (fp16): input and output once, the weight once."""
    return 2 * P * k * k * ci * co, 2 * (P * ci + P * co + k * k * ci * co + co)


def adapter_cost(H: int, W: int, batch: int = 1, in_channels: int = 3, channels=(320, 640, 1280, 1280),
                 num_res_blocks: int = 2):
    """(FLOPs, bytes) of one full_adapter_xl forward at an H x W image, counted as diffusers' layers (the average pool
    and the 1x1 in_conv as such, not the 9-tap folded conv the native adapter launches; the pool's adds are left
    out).  Bytes: each layer reads its input and writes its output once, the resnet's 1x1 block2 also reads the skip,
    the weights once; the image is read once by the unshuffle, which writes the unshuffled NHWC copy."""
    c = channels
    P = (H // 16) * (W // 16)
    f = b = 0

    def add(cost, extra=0):
        nonlocal f, b
        f, b = f + cost[0], b + cost[1] + extra

    b += 2 * 2 * in_channels * H * W                             # unshuffle: read the image, write the NHWC copy
    add(_conv(P, in_channels * 256, c[0]))                       # conv_in
    for i, co in enumerate(c):
        if i == 1:
            add(_conv(P, c[0], c[1], k=1))                       # in_conv 1x1
        if i == 2:
            b += 2 * (P * c[1] + P // 4 * c[1])                  # AvgPool2d(2)
            P //= 4
            add(_conv(P, c[1], c[2], k=1))
        for _ in range(num_res_blocks):
            add(_conv(P, co, co))                                # block1 (+ ReLU)
            add(_conv(P, co, co, k=1), 2 * P * co)               # block2 + the skip
    return batch * f, batch * b


def injection_bytes(H: int, W: int, batch: int = 1, cfg: bool = True, channels=(320, 640, 1280, 1280)) -> int:
    """Algorithmic bytes of one step's feature injection: at each of the 4 points every row of each CFG half reads
    its skip and the feature and writes the skip (fp16)."""
    h, w = H // 16, W // 16
    elems = h * w * channels[0] + h * w * channels[1] + (h // 2) * (w // 2) * (channels[2] + channels[3])
    return 3 * 2 * elems * batch * (2 if cfg else 1)


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


def _emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools_out"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_t2i_adapter.py needs a GPU")
    from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET, SDXL_T2I_ADAPTER
    from imagharmony_b200.controlnet import ControlNetModel
    from imagharmony_b200.weights import random_module
    from ip_adapter.custom_pipelines import StableDiffusionXLAdapterPipeline, StableDiffusionXLControlNetPipeline
    from tools.bench_img2img import card
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda"
    gpu = card()
    rows = []
    pipe = StableDiffusionXLAdapterPipeline.from_random(SDXL_BASE, SDXL_T2I_ADAPTER, seed=0, device=dev)
    g = torch.Generator("cpu").manual_seed(0)

    # ---- the adapter forward at every bucket
    for H, W in BUCKETS:
        for B in (1, 4):
            x = torch.rand(B, 3, H, W, generator=g).half().to(dev)
            ts = _time_ms(lambda: pipe.adapter(x), args.warmup, args.iters)
            fl, by = adapter_cost(H, W, B)
            ms = statistics.median(ts)
            _emit(rows, {"card": gpu, "what": "adapter_forward", "height": H, "width": W, "batch": B, "ms": ms,
                         "spread_ms": max(ts) - min(ts), "gflop": fl / 1e9, "mbytes": by / 1e6,
                         "tflops": fl / ms / 1e9, **bound(fl, by)})
            del x

    # ---- the 1024^2 CFG step with and without the adapter: the engine's two captured graphs, alternated
    D, P = SDXL_BASE.cross_attention_dim, SDXL_BASE.pooled_embed_dim
    emb = dict(prompt_embeds=torch.randn(1, 77, D, generator=g).half(),
               negative_prompt_embeds=torch.randn(1, 77, D, generator=g).half(),
               pooled_prompt_embeds=torch.randn(1, P, generator=g).half(),
               negative_pooled_prompt_embeds=torch.randn(1, P, generator=g).half())
    sketch = torch.rand(1, 3, 1024, 1024, generator=g)
    # a schedule one step longer than a round: every replay of a round reads an index inside the schedule's tables
    T = args.replays + 1
    pipe(image=sketch, num_inference_steps=T, adapter_conditioning_factor=0.5, output_type="latent", **emb)
    eng, loop = pipe.engine, pipe.engine._loop
    graphs = {k.adapter: gr for k, (gr, _) in eng._graphs.items() if (k.n, k.h, k.w, k.T) == (1, 128, 128, T)}
    assert set(graphs) == {False, True}, list(eng._graphs)
    lat0 = (torch.randn(1, 4, 128, 128, generator=g) * pipe.scheduler.init_noise_sigma).half().to(dev)
    per = {False: [], True: []}
    for r in range(args.rounds + 1):                               # round 0 warms both graphs up, untimed
        for flag in ((False, True) if r % 2 == 0 else (True, False)):
            eng._restart(loop, lat0, 0)                             # the loop's start: latents, step 0, first input
            ts = _time_ms(lambda: [graphs[flag].replay() for _ in range(args.replays)], 0, 1)
            if r:
                per[flag].append(ts[0] / args.replays)
    step = {"card": gpu, "what": "cfg_step_1024", "replays_per_round": args.replays, "rounds": args.rounds,
            "plain_ms": statistics.median(per[False]), "plain_spread_ms": max(per[False]) - min(per[False]),
            "adapter_ms": statistics.median(per[True]), "adapter_spread_ms": max(per[True]) - min(per[True]),
            "injection_mbytes": injection_bytes(1024, 1024) / 1e6}
    step["delta_ms"] = step["adapter_ms"] - step["plain_ms"]
    step["delta_within_spread"] = abs(step["delta_ms"]) <= max(step["plain_spread_ms"], step["adapter_spread_ms"])
    _emit(rows, step)

    # ---- one whole call with the adapter against the same call with one ControlNet
    cn = StableDiffusionXLControlNetPipeline(pipe.unet, random_module(ControlNetModel, SDXL_CONTROLNET, 23, dev))
    calls = {"adapter": lambda: pipe(image=sketch, num_inference_steps=args.steps, output_type="latent", **emb),
             "controlnet": lambda: cn(image=sketch, num_inference_steps=args.steps, output_type="latent", **emb)}
    call = {"card": gpu, "what": f"call_{args.steps}_steps_1024", "batch": 1}
    for name, fn in calls.items():
        ts = _time_ms(fn, 1, max(2, args.iters // 2))
        call[f"{name}_ms"] = statistics.median(ts)
        call[f"{name}_spread_ms"] = max(ts) - min(ts)
    call["controlnet_over_adapter"] = call["controlnet_ms"] / call["adapter_ms"]
    _emit(rows, call)
    with open(os.path.join(args.out, "bench_t2i_adapter.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
