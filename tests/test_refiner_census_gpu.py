"""Per-call census of the SDXL refiner UNet (random weights, text-only cross-attention over 77 tokens) at every SDXL
bucket with one image and CFG, at 1024^2 with 2, 4 and 8 images, and once without CFG: every op call is compared with
its reference at its real shape against the bar tests/census.py derives (the plan, bucket list and report of
test_unet_census_gpu.py).  The refiner reaches shapes the base does not: 384 / 768 / 1536-channel convs and GEMMs
(1152 / 2304 / 3072 channels on the skip concatenations), GroupNorm groups of 12 to 96 channels, 6 / 12 / 24-head
attention, K = 1280 cross-attention projections, and a fourth level of 16 x 16 latents at 1024^2.  `-s` also prints
the GEMM launches of that level (M = 512 rows per image pair) with their `tile_n` argument (0: the library's automatic
tile choice) and err / bar."""
import pytest
import torch

import census
from test_kernels_gpu import ops  # noqa: F401  (fixture: TF32 off for the fp32 references)
from test_unet_census_gpu import BUCKETS, _finish, plan

pytestmark = pytest.mark.gpu

CASES = ([(h, w, 1, True) for h, w in BUCKETS] + [(1024, 1024, n, True) for n in (2, 4, 8)]
         + [(1024, 1024, 1, False)])


@pytest.fixture(scope="module")
def refiner_unet(ops):  # noqa: F811
    import bench
    from imagharmony_b200.config import SDXL_REFINER
    return bench.build_native(SDXL_REFINER, "cuda")


@pytest.mark.parametrize("height,width,n,cfg", CASES,
                         ids=[f"{h}x{w}-n{n}{'' if c else '-nocfg'}" for h, w, n, c in CASES])
def test_refiner_unet_census(ops, refiner_unet, monkeypatch, height, width, n, cfg):  # noqa: F811
    unet = refiner_unet
    ucfg = unet.config
    B = 2 * n if cfg else n
    g = torch.Generator("cpu").manual_seed(height * 5 + width + n)
    sample = torch.randn(B, 4, height // 8, width // 8, generator=g).half().cuda()
    ehs = torch.randn(B, 77, ucfg.cross_attention_dim, generator=g).half().cuda()
    te = torch.randn(B, ucfg.pooled_embed_dim, generator=g).half().cuda()
    tid = torch.tensor([[height, width, 0., 0., 6.0]] * B, device="cuda")
    bench_workload = (height, width, n, cfg) == (1024, 1024, 1, True)
    c = census.Census(ops, check_all=bench_workload, plan=plan).install(monkeypatch)
    with torch.no_grad():
        out = unet(sample, torch.full((B,), 201.0, device="cuda"), ehs, te, tid)
    monkeypatch.undo()
    assert out.shape == (B, 4, height // 8, width // 8)
    attn = [r["shape"] for r in c.rows.values() if r["op"] == "attention"]
    assert attn and all(s.endswith("n_ip=0") for s in attn), attn
    cross = {s.split()[2] for s in attn if s.split()[2].split("x")[0] != s.split()[2].split("x")[1]}
    assert cross and all(qk.split("x")[1] == "77" for qk in cross), cross
    if bench_workload:
        rows = B * (height // 64) * (width // 64)
        print(f"\n== GEMM launches of the {height // 64}x{width // 64} level (M = {rows}):")
        for r in sorted(c.rows.values(), key=lambda r: r["shape"]):
            if r["op"] == "linear" and r["shape"].startswith(f"{rows}x"):
                print(f"   {r['shape']}  calls {r['calls']}  err/bar {r['worst']:.3f}")
    _finish(c, f"refiner UNet {height}x{width} n={n} cfg={cfg} (batch {B})")
