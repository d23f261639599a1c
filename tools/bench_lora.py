"""Cost of a merged SDXL LoRA on one GPU.

    python tools/bench_lora.py [--ranks 64 128] [--rounds 7] [--replays 10] [--out tools_out]

Writes a synthetic full-coverage LoRA for the SDXL-base UNet (every targetable module, kohya keys, `.alpha` = r / 2)
per rank under the output directory as .safetensors, then on a random-init SDXL-base pipeline with its IP processors:
  load_ms        : load_lora_weights, split into file read (host), merge GEMMs (CUDA events around the merge launches,
                   with their algorithmic FLOPs 2 N r_pad K' and bytes: up, down, original read, merged weight written)
                   and re-derivation (UNet.finalize(), host clock after a synchronise)
  set_ms         : set_adapters with another weight (merge + re-derivation)
  recapture_ms   : the first 1024^2 CFG denoise call after the change against a repeat call (host clock, synchronised)
  step_ms        : the SDXL 1024^2 CFG step graph without and with the LoRA, `rounds` alternated rounds of `replays`
                   graph replays each, CUDA events; median and spread (max - min) per side
  kept_bytes     : the device memory of the originals kept for unload / re-merge
Prints one JSON line per rank and writes them to <out>/bench_lora.json.  The card's name, power limit and max SM clock
are read in the same process and reported with the numbers.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.bench_img2img import card  # noqa: E402


def synthetic_lora(unet, rank: int, seed: int = 0):
    """kohya state dict covering every targetable module, deltas about 0.1 |W|."""
    from imagharmony_b200.lora import unet_name_table
    from lora_ref import module_shapes, random_lora, to_kohya
    table = unet_name_table(unet)
    return to_kohya(random_lora(module_shapes(unet, table), rank, seed, alpha=rank / 2), "unet", table)


def merge_cost(lw) -> dict:
    """Algorithmic FLOPs and bytes of one merge of every loaded term (fp16 operands)."""
    flops = byts = 0
    for ad in lw.adapters.values():
        for comp, mods in ad.terms.items():
            for mod, t in mods.items():
                N, rp = t.up.shape
                K = t.down_t.shape[0]
                flops += 2 * N * rp * K
                byts += 2 * (N * rp + K * rp + 2 * N * K)
    return {"merge_gflop": flops / 1e9, "merge_gbytes": byts / 1e9}


def timed_events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools_out"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora.py needs a GPU")
    from safetensors.torch import save_file
    import imagharmony_b200.lora as L
    from imagharmony_b200.config import SDXL_BASE
    from imagharmony_b200.denoise import DenoiseEngine
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline

    os.makedirs(args.out, exist_ok=True)
    pipe = StableDiffusionXLCustomPipeline.from_random(SDXL_BASE, seed=0)
    unet = pipe.unet
    cfg = unet.config
    g = torch.Generator("cpu").manual_seed(1)
    ehs = torch.randn(2, 77 + cfg.num_ip_tokens, cfg.cross_attention_dim, generator=g).half()
    pooled = torch.randn(2, cfg.pooled_embed_dim, generator=g).half()
    tid = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]])
    lat = torch.randn(1, 4, 128, 128, generator=g).half().pin_memory()
    eng = DenoiseEngine(unet)

    def call(steps):
        return eng.run(lat, ehs[1:], ehs[:1], pooled[1:], pooled[:1], tid, steps, guidance_scale=5.0, ip_scale=1.0)

    def step_graph_ms():
        call(args.replays)                        # captured graphs for this state
        return timed_events(lambda: call(args.replays)) / args.replays

    results = []
    for rank in args.ranks:
        path = os.path.join(args.out, f"sdxl_lora_r{rank}.safetensors")
        save_file({k: v.half().contiguous() for k, v in synthetic_lora(unet, rank).items()}, path)
        row = {"card": card(), "rank": rank, "file_mb": os.path.getsize(path) / 2 ** 20}
        # load: file read / merge GEMMs / re-derivation, measured piece by piece around the same calls load makes
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sd = L.read_state_dict(path)
        row["read_ms"] = (time.perf_counter() - t0) * 1e3
        fin = unet.finalize
        fin_ms = []

        def timed_finalize():
            torch.cuda.synchronize()
            t = time.perf_counter()
            fin()
            torch.cuda.synchronize()
            fin_ms.append((time.perf_counter() - t) * 1e3)
        merge_ms = []
        sync = L.LoraWeights.sync

        def timed_sync(self, comp, factors):
            if comp != L.UNET:
                return sync(self, comp, factors)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            self.unet.finalize = lambda: None
            try:
                n = sync(self, comp, factors)
            finally:
                del self.unet.finalize
            b.record()
            torch.cuda.synchronize()
            merge_ms.append(a.elapsed_time(b))
            if n:
                timed_finalize()
            return n
        L.LoraWeights.sync = timed_sync
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.load_lora_weights(sd, adapter_name="bench")
            torch.cuda.synchronize()
            row["load_total_ms"] = (time.perf_counter() - t0) * 1e3 + row["read_ms"]
            row["merge_ms"], row["rederive_ms"] = merge_ms[-1], fin_ms[-1]
            row.update(merge_cost(pipe._lora))
            row["merge_tflops"] = row["merge_gflop"] / row["merge_ms"]
            row["merge_tbytes_s"] = row["merge_gbytes"] / row["merge_ms"]
            merge_ms.clear(), fin_ms.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.set_adapters("bench", 0.5)
            torch.cuda.synchronize()
            row["set_adapters_ms"] = (time.perf_counter() - t0) * 1e3
            row["set_adapters_merge_ms"], row["set_adapters_rederive_ms"] = merge_ms[-1], fin_ms[-1]
        finally:
            L.LoraWeights.sync = sync
        row["kept_mb"] = pipe._lora.kept_bytes() / 2 ** 20
        # first call after the change (graph capture) against a repeat
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call(2)
        torch.cuda.synchronize()
        first = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        call(2)
        torch.cuda.synchronize()
        row["recapture_ms"] = first - (time.perf_counter() - t0) * 1e3
        # step graph with and without the LoRA, alternated
        with_l, without = [], []
        for _ in range(args.rounds):
            pipe.disable_lora()
            without.append(step_graph_ms())
            pipe.enable_lora()
            with_l.append(step_graph_ms())
        for k, v in (("step_ms_base", without), ("step_ms_lora", with_l)):
            row[k] = statistics.median(v)
            row[k + "_spread"] = max(v) - min(v)
        pipe.unload_lora_weights()
        del sd
        results.append(row)
        print(json.dumps(row), flush=True)
    with open(os.path.join(args.out, "bench_lora.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
