"""HarmonyBench-shape sweep (BASELINE config 5): {512, 768, 1024}^2 x steps {20, 50} x images {1, 4, 16} per GPU ->
denoise-steps/s, ms/step, algorithmic TFLOP/s, fraction of the sustained tensor peak.  Run alone for one GPU, or under
`python -m torch.distributed.run --nproc-per-node N tools/sweep.py` for the N-GPU weak-scaling rows (independent images
per rank, barrier + CUDA events, max over ranks -- the path has no per-step collective).
Writes tools_out/sweep_n{N}.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from imagharmony_b200.config import SDXL_BASE as cfg  # noqa: E402
from imagharmony_b200.denoise import DenoiseEngine  # noqa: E402


def main():
    rank, local, world = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("LOCAL_RANK", "0"), ("WORLD_SIZE", "1")))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    images = [int(x) for x in os.environ.get("IH_SWEEP_IMAGES", "1,4,16").split(",")]
    steps = [int(x) for x in os.environ.get("IH_SWEEP_STEPS", "20,50").split(",")]
    unet = bench.build_native(cfg, dev)
    eng = DenoiseEngine(unet)
    pk = bench.peaks()
    rows = []
    for res in (512, 768, 1024):
        for n in images:
            lat = res // 8
            for K in steps:
                ins = [t.pin_memory() for t in bench.synth_inputs(cfg, n, lat, K, rank)]
                eng.run(*ins, K, stop_after=3)
                if dist is not None:
                    dist.barrier()
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                eng.run(*ins, K)
                e.record()
                torch.cuda.synchronize()
                sec = s.elapsed_time(e) * 1e-3
                if dist is not None:
                    t = torch.tensor([sec], device=dev, dtype=torch.float64)
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                    sec = float(t[0])
                tf = bench.TFLOP_PER_PAIR.get(lat, 13.524 * (lat / 128.0) ** 2) * n
                rows.append({"gpus": world, "res": res, "images_per_gpu": n, "unet_batch": 2 * n, "steps": K,
                             "ms_per_step": sec / K * 1e3, "denoise_steps_per_s": world * n * K / sec,
                             "tflops_per_gpu": tf * K / sec, "frac_sustained_peak": tf * K / sec / pk["tflops_sustained"]})
                if rank == 0:
                    print(json.dumps(rows[-1]), flush=True)
            eng.invalidate_graphs()
            eng._pool.clear()
            torch.cuda.empty_cache()
    if rank == 0:
        os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
        json.dump(rows, open(os.path.join(ROOT, "tools_out", f"sweep_n{world}.json"), "w"), indent=1)
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
