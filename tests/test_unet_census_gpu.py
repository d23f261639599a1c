"""Per-call census of the SDXL-base UNet (with its IP-Adapter processors, n_ip = 4) and the SDXL VAE decoder at the
resolutions SDXL is used at: every SDXL aspect-ratio bucket plus 512^2 and 768^2, 1 to 8 images per call with CFG and
one call without.  The execution plan of a kernel follows the shape (GEMM tile width, conv spatial tile, attention
KV-split plan, GroupNorm block mapping), so these calls reach token counts, tile remainders and wave remainders that
the hand-picked shapes of the kernel tests do not.

Each op call is compared with a reference computed from its own inputs (tests/census.py: references and the
derivation of every bar), so an error of a few ulps in one layer at one shape shows up directly instead of under the
fp16 error the whole forward accumulates.  The bench workload (1024^2, one image, CFG) checks every call; elsewhere
the first call of each distinct key (op, tensor shapes and strides, flags, tile_n, stride, n_ip, KV-split workspace or
not).  Random weights, eager forwards (graph replay is bit-identical to eager, test_unet_gpu.py).  `-s` prints one row
per key and, at the end, how many distinct attention split plans, conv tiles and GroupNorm configurations ran."""
import pytest
import torch

import census
from test_kernels_gpu import ops  # noqa: F401  (fixture: TF32 off for the fp32 references)

pytestmark = pytest.mark.gpu

BUCKETS = [(1024, 1024), (1152, 896), (896, 1152), (1216, 832), (832, 1216), (1344, 768), (768, 1344), (1536, 640),
           (640, 1536), (512, 512), (768, 768)]
UNET_CASES = ([(h, w, 1, True) for h, w in BUCKETS] + [(1024, 1024, n, True) for n in (2, 4, 8)]
              + [(832, 1216, n, True) for n in (2, 4, 8)] + [(1024, 1024, 1, False)])
COVERED = {"attention split plans": set(), "conv spatial tiles": set(), "GroupNorm configurations": set()}


def conv_tile(Ho, Wo):
    """bw x bh of the implicit-GEMM conv: a restatement of the tile choice in gemm.cu conv_impl ("spatial tile: bw x bh =
    128 output pixels, minimise padded tiles"; 128 output pixels, fewest tiles, widest first), which the library does
    not report.  It labels the census rows and counts the tiles covered; keep it in step with conv_impl."""
    best = None
    for bw in (128, 64, 32, 16, 8, 4, 2, 1):
        t = -(-Wo // bw) * -(-Ho // (128 // bw))
        if best is None or t < best[0]:
            best = (t, bw)
    return best[1], 128 // best[1]


def plan(name, p):
    """Plan part of the census key: whether an attention call gets a KV-split workspace (and its size, which follows
    the split plan), the conv's spatial tile."""
    from imagharmony_b200 import _lib
    if name == "attention":
        ws = int(_lib.load().ih_attention_workspace_bytes(p["B"], p["H"], p["Nq"], p["Nk"], p["n_ip"])) if p["kv_split"] else 0
        if ws:
            COVERED["attention split plans"].add((p["B"], p["H"], p["Nq"], p["Nk"], ws))
        return f"ws{ws}" if ws else "whole"
    if name == "conv3x3":
        B, H, W, _ = p["x"].shape
        bw, bh = conv_tile(H // p["stride"], W // p["stride"])
        COVERED["conv spatial tiles"].add((bw, bh))
        return f"tile{bw}x{bh}"
    if name == "groupnorm":
        B, H, W, C0 = p["x0"].shape
        COVERED["GroupNorm configurations"].add((B, H * W, C0 + (0 if p["x1"] is None else p["x1"].shape[-1]),
                                                 p["groups"]))
    return None


@pytest.fixture(scope="module", autouse=True)
def coverage_summary():
    yield
    print("\n== census coverage: " + ", ".join(f"{len(v)} {k}" for k, v in COVERED.items()))


@pytest.fixture(scope="module")
def sdxl_unet(ops):  # noqa: F811
    import bench
    from imagharmony_b200.config import SDXL_BASE
    return bench.build_native(SDXL_BASE, "cuda")


@pytest.fixture(scope="module")
def sdxl_vae(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_VAE
    from imagharmony_b200.vae import AutoencoderKLDecoder
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(AutoencoderKLDecoder(SDXL_VAE))
    return AutoencoderKLDecoder.from_state_dict(SDXL_VAE, random_state_dict(shapes, 2, device="cuda"), device="cuda")


def _finish(c, title):
    torch.cuda.synchronize()
    print("\n" + c.report(title))
    assert not c.unread(), f"{title}: arguments no reference reads: {c.unread()}"
    bad = c.failures()
    assert not bad, f"{title}: {len(bad)} keys beyond their bar:\n" + "\n".join(
        f"{r['op']} {r['shape']} {r['plan']}: err/bar {r['worst']:.3f}" for r in bad)


@pytest.mark.parametrize("height,width,n,cfg", UNET_CASES,
                         ids=[f"{h}x{w}-n{n}{'' if c else '-nocfg'}" for h, w, n, c in UNET_CASES])
def test_unet_census(ops, sdxl_unet, monkeypatch, height, width, n, cfg):  # noqa: F811
    unet = sdxl_unet
    ucfg = unet.config
    B = 2 * n if cfg else n
    g = torch.Generator("cpu").manual_seed(height * 7 + width + n)
    sample = torch.randn(B, 4, height // 8, width // 8, generator=g).half().cuda()
    ehs = torch.randn(B, 77 + ucfg.num_ip_tokens, ucfg.cross_attention_dim, generator=g).half().cuda()
    te = torch.randn(B, ucfg.pooled_embed_dim, generator=g).half().cuda()
    tid = torch.tensor([[height, width, 0., 0., height, width]] * B, device="cuda")
    bench_workload = (height, width, n, cfg) == (1024, 1024, 1, True)
    c = census.Census(ops, check_all=bench_workload, plan=plan).install(monkeypatch)
    with torch.no_grad():
        out = unet(sample, torch.full((B,), 501.0, device="cuda"), ehs, te, tid)
    monkeypatch.undo()
    assert out.shape == (B, 4, height // 8, width // 8)
    ips = {r["shape"] for r in c.rows.values() if r["op"] == "attention" and "n_ip=4" in r["shape"]}
    assert ips, "the IP-Adapter layers must run their decoupled attention"
    _finish(c, f"UNet {height}x{width} n={n} cfg={cfg} (batch {B})")


@pytest.mark.parametrize("height,width", BUCKETS, ids=[f"{h}x{w}" for h, w in BUCKETS])
def test_vae_decoder_census(ops, sdxl_vae, monkeypatch, height, width):  # noqa: F811
    g = torch.Generator("cpu").manual_seed(height + width)
    z = torch.randn(1, 4, height // 8, width // 8, generator=g).half().cuda()
    c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
    img = sdxl_vae.decode(z)
    monkeypatch.undo()
    assert img.shape == (1, 3, height, width)
    ops_run = {(r["op"], "alpha=" in r["shape"]) for r in c.rows.values()}
    assert {("softmax_rows_masked_", False), ("conv3x3", True), ("linear", True)} <= ops_run   # the scaled stream
    _finish(c, f"VAE decoder {height}x{width}")
