"""Ramp breakdown of one GEMM launch inside a dependent chain (globaltimer stamps of CTA 0).  `python
tools/gemm_trace.py pp` traces the ping-pong kernel at the q|k|v and GEGLU launches of a 1024^2 step."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from imagharmony_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
buf = torch.zeros(16, dtype=torch.int64, device="cuda")
names = ["entry", "setup done", "pdl_wait done", "first operands", "acc0 ready", "acc1 ready", "acc2 ready", "acc3+ ready", "cta done",
         "slab0 in regs", "slab0 in smem", "slab1/mid in smem", "last slab in smem", "stores read out"]


def run(label, M, N, K, geglu=False, tn=0, full=False):
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
    g = torch.ones(K, device="cuda").half()
    kw = {}
    if full:
        kw = dict(bias=torch.randn(N, device="cuda").half(), residual=torch.randn(M, N, device="cuda").half(),
                  stats_out=torch.empty((N // 64, M, 2), dtype=torch.float32, device="cuda"))
    for _ in range(3):
        n = ops.layernorm(x, g, g)
        ops.linear(n, w, geglu=geglu, tile_n=tn, **kw)
    torch.cuda.synchronize()
    lib.ih_gemm_set_trace(buf.data_ptr())
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = ops.layernorm(x, g, g)
    s.record()
    ops.linear(n, w, geglu=geglu, tile_n=tn, **kw)
    e.record()
    torch.cuda.synchronize()
    lib.ih_gemm_set_trace(None)
    t = buf.cpu().tolist()
    rel = [(t[i] - t[0]) / 1e3 if t[i] else None for i in range(14)]
    print(label, f"event {s.elapsed_time(e) * 1e3:.1f} us |", ", ".join(f"{n}={v:.2f}" for n, v in zip(names, rel) if v is not None))
    buf.zero_()


def run_pp(label, M, C, geglu):
    """One LayerNorm-folded q|k|v (N = 3C) or GEGLU (N = 8C) launch with bias on the ping-pong kernel.  CTA 0's stamps
    give the accumulator-ready times of its first three tiles (warpgroups 1, 2, 1) and of its last; from the second tile
    on the main loops run back to back, so the gap between consecutive ready stamps is one tile's main loop."""
    N = 8 * C if geglu else 3 * C
    x = torch.randn(M, C, device="cuda").half()
    w = (torch.randn(N, C, device="cuda") * C ** -0.5).half()
    b = torch.randn(N, device="cuda").half()
    st = torch.rand((C // 64, M, 2), device="cuda")
    st[..., 1] += 64.0
    for _ in range(3):
        ops.linear(x, w, b, geglu=geglu, ln=(st, 1e-5), tile_n=ops.TILE_PINGPONG)
    torch.cuda.synchronize()
    lib.ih_gemm_set_trace(buf.data_ptr())
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    ops.linear(x, w, b, geglu=geglu, ln=(st, 1e-5), tile_n=ops.TILE_PINGPONG)
    e.record()
    torch.cuda.synchronize()
    lib.ih_gemm_set_trace(None)
    t = [(v - buf[0].item()) / 1e3 for v in buf.cpu().tolist()[:9]]
    buf.zero_()
    kb = C // 64
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-M // 128) * -(-(N // 2 if geglu else N) // (64 if geglu else 128))
    loops = [t[5] - t[4], t[6] - t[5]]
    print(f"{label} M{M} N{N} K{C}: kb {kb}, tiles/SM {tiles / sms:.2f}, event {s.elapsed_time(e) * 1e3:.1f} us | "
          f"first stage {t[3]:.2f}, tile 0 ready {t[4]:.2f}, main loops of tiles 1, 2 "
          f"{loops[0]:.2f}, {loops[1]:.2f} us ({sum(loops) / (2 * kb):.3f} us per k-block), last tile ready {t[7]:.2f}, "
          f"cta done {t[8]:.2f}", flush=True)


if len(sys.argv) > 1 and sys.argv[1] == "pp":
    # the ping-pong launches of a 1024^2 step with CFG (batch 2): level 1 (res / 16, C 640), level 2 (res / 32, C 1280)
    for lvl, (M, C) in enumerate([(2 * 64 * 64, 640), (2 * 32 * 32, 1280)], 1):
        for geglu in (False, True):
            run_pp(f"level {lvl} {'GEGLU' if geglu else 'q|k|v'}", M, C, geglu)
    sys.exit(0)

run("1 tile 128x256x64      ", 128, 256, 64, tn=256)
run("1280^2 (80 tiles)      ", 2048, 1280, 1280, tn=256)
run("1280^2 auto (112 tiles) ", 2048, 1280, 1280, tn=0)
run("1280^2 auto +bias+res+stats", 2048, 1280, 1280, tn=0, full=True)
run("1280^2 bn128 (160 tiles)", 2048, 1280, 1280, tn=128)
run("QKV 2048x3840x1280     ", 2048, 3840, 1280, tn=256)
run("FF-in geglu            ", 2048, 10240, 1280, geglu=True, tn=256)
run("FF-out 2048x1280x5120  ", 2048, 1280, 5120, tn=256)
run("FF-in geglu pair       ", 2048, 10240, 1280, geglu=True, tn=512)
