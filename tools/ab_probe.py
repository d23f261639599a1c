"""Small A/B probes (graph-timed, same process => same thermal state).  `python tools/ab_probe.py tile` measures the
main-loop cost per 64-deep k-block of the 128xBN tiles, plain and GEGLU, with every SM busy (calibrates the tile
costs in gemm.cu).  `python tools/ab_probe.py pp` times the ping-pong kernel against gemm_f16_kernel at the
LayerNorm-folded q|k|v and GEGLU launches of the SDXL base and refiner UNets (calibrates pick_pp in gemm.cu)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from imagharmony_b200 import ops  # noqa: E402
from tools.microbench import timeit, r  # noqa: E402


def tile_costs():
    M = 2048
    cols = torch.cuda.get_device_properties(0).multi_processor_count // 16
    for bn in (128, 160, 192, 256):
        N = cols * bn                   # cols x 16 tiles <= #SMs: one round with (nearly) every SM busy
        ts = []
        for K in (1280, 5120):
            x, w = r(M, K), r(N, K, scale=K ** -0.5)
            ts.append(timeit(lambda: ops.linear(x, w, tile_n=bn)))
        per_kb = (ts[1] - ts[0]) / ((5120 - 1280) / 64)
        print(f"128x{bn}: K=1280 {ts[0]*1e6:.1f} us, K=5120 {ts[1]*1e6:.1f} us -> {per_kb*1e6:.3f} us per k-block, "
              f"fixed {(ts[0] - 20 * per_kb)*1e6:.1f} us", flush=True)


def geglu_tile_costs():
    """The same for GEGLU (value + gate halves in one B tile of `bn` rows, bn / 2 outputs), LayerNorm-folded with bias
    as in the UNet's feed-forward: one round with (nearly) every SM busy."""
    M = 2048
    cols = torch.cuda.get_device_properties(0).multi_processor_count // 16
    for bn in (128, 192, 256):
        N = 2 * cols * (bn // 2)
        ts = []
        for K in (1280, 5120):
            x, w, b = r(M, K), r(N, K, scale=K ** -0.5), r(N)
            st = torch.rand((K // 64, M, 2), device="cuda")
            st[..., 1] += 64.0
            ts.append(timeit(lambda: ops.linear(x, w, b, geglu=True, ln=(st, 1e-5), tile_n=bn)))
        per_kb = (ts[1] - ts[0]) / ((5120 - 1280) / 64)
        print(f"GEGLU 128x{bn}: K=1280 {ts[0]*1e6:.1f} us, K=5120 {ts[1]*1e6:.1f} us -> {per_kb*1e6:.3f} us per k-block, "
              f"fixed {(ts[0] - 20 * per_kb)*1e6:.1f} us", flush=True)


def geglu_shapes():
    """The UNet's LayerNorm-folded GEGLU launches at 1024^2, batch 2 (level 2: M 2048, K 1280; level 1: M 8192, K 640)
    on every GEGLU tile and on the library's choice."""
    for (M, K) in [(2048, 1280), (8192, 640)]:
        N = 8 * K
        x, w, b = r(M, K), r(N, K, scale=K ** -0.5), r(N)
        st = torch.rand((K // 64, M, 2), device="cuda")
        st[..., 1] += 64.0
        for bn in (128, 192, 256, 0):
            t = timeit(lambda: ops.linear(x, w, b, geglu=True, ln=(st, 1e-5), tile_n=bn))
            print(f"GEGLU M{M} N{N} K{K} bn{bn}: {t*1e6:.1f} us", flush=True)


def shapes():
    for (M, N, K, geglu, tn) in [(2048, 1280, 1280, False, 0), (2048, 3840, 1280, False, 0), (8192, 1920, 640, False, 0),
                                 (2048, 10240, 1280, True, 0), (2048, 1280, 5120, False, 0)]:
        x, w, b = r(M, K), r(N, K, scale=K ** -0.5), r(N)
        t = timeit(lambda: ops.linear(x, w, b, geglu=geglu, tile_n=tn))
        print(f"gemm M{M} N{N} K{K} g{int(geglu)}: {t*1e6:.1f} us", flush=True)
    for (B, H, Cin, Cout, s) in [(2, 32, 1280, 1280, 1), (2, 64, 640, 640, 1), (2, 128, 320, 320, 1), (2, 32, 2560, 1280, 1),
                                 (2, 64, 1920, 640, 1)]:
        x = r(B, H, H, Cin)
        w = r(Cout, 9 * Cin, scale=(9 * Cin) ** -0.5)
        b = r(Cout)
        for tn in (128, 192, 256, 0):
            t = timeit(lambda: ops.conv3x3(x, w, b, stride=s, tile_n=tn))
            print(f"conv B{B} {H}^2 {Cin}->{Cout} bn{tn}: {t*1e6:.1f} us", flush=True)


def pp_shapes():
    """LayerNorm-folded q|k|v (N = 3C) and GEGLU (N = 8C) launches with bias, as in the UNet: M = 2 * images * tokens
    (CFG), C the block width.  The base UNet's transformer levels have C = 640 at res / 16 and C = 1280 at res / 32,
    the refiner's C = 768 and 1536 at the same levels.  `old` is gemm_f16_kernel's fastest tile (GEGLU: the 256-row
    tile, its automatic choice), `auto` the library's choice."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"{torch.cuda.get_device_name(0)}, {sms} SMs", flush=True)
    for net, widths in (("base", (640, 1280)), ("refiner", (768, 1536))):
        for res in (512, 768, 1024):
            for images in (1, 4):
                for lvl, c in enumerate(widths):
                    m = 2 * images * (res // (16 << lvl)) ** 2
                    st = torch.rand((c // 64, m, 2), device="cuda")
                    st[..., 1] += 64.0
                    x = r(m, c)
                    for geglu in (False, True):
                        n = 8 * c if geglu else 3 * c
                        w, b = r(n, c, scale=c ** -0.5), r(n)

                        def run(tn):
                            return timeit(lambda: ops.linear(x, w, b, geglu=geglu, ln=(st, 1e-5), tile_n=tn))
                        old_tiles = (256,) if geglu else (128, 160, 192, 256)
                        old = min(run(tn) for tn in old_tiles)
                        pp, auto = run(ops.TILE_PINGPONG), run(0)
                        kb = (c + 63) // 64
                        tiles = -(-m // 128) * -(-(n // 2 if geglu else n) // (64 if geglu else 128))
                        print(f"{net} {res}^2 x{images} C{c} {'GEGLU' if geglu else 'qkv  '} M{m} N{n} K{c}: kb {kb}, "
                              f"pp tiles/SM {tiles / sms:.2f}: old {old*1e6:.1f} us, pp {pp*1e6:.1f} us "
                              f"(x{old / pp:.3f}), auto {auto*1e6:.1f} us", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "tile":
        tile_costs()
        geglu_tile_costs()
    elif len(sys.argv) > 1 and sys.argv[1] == "geglu":
        geglu_shapes()
    elif len(sys.argv) > 1 and sys.argv[1] == "pp":
        pp_shapes()
    else:
        shapes()
