"""Per-call census (tests/census.py) of the SDXL T2I-Adapter forward at every SDXL bucket, batch 1, and at 1024^2 with
4 images: conv_in and every block1 on the implicit-GEMM conv (block1 with the ReLU epilogue), block2 + the skip and
block 1's in_conv on the GEMM, block 2's folded average pool + in_conv on the bottom/right-padded stride-2 conv.  Random
weights; every call is checked at 1024^2 with one image, the first call of each distinct key elsewhere."""
import zlib

import pytest
import torch

import census
from test_kernels_gpu import ops  # noqa: F401  (fixture: TF32 off for the fp32 references)
from test_unet_census_gpu import BUCKETS, _finish, plan

pytestmark = pytest.mark.gpu

CASES = [(h, w, 1) for h, w in BUCKETS] + [(1024, 1024, 4)]


@pytest.fixture(scope="module")
def sdxl_adapter(ops):  # noqa: F811
    from imagharmony_b200.config import SDXL_T2I_ADAPTER
    from imagharmony_b200.t2i_adapter import T2IAdapter
    return T2IAdapter.from_random(SDXL_T2I_ADAPTER, seed=41, device="cuda")


@pytest.mark.parametrize("height,width,n", CASES, ids=[f"{h}x{w}-n{n}" for h, w, n in CASES])
def test_t2i_adapter_census(ops, sdxl_adapter, monkeypatch, height, width, n):  # noqa: F811
    g = torch.Generator("cpu").manual_seed(zlib.crc32(repr(("t2i", height, width, n)).encode()))
    x = torch.rand(n, 3, height, width, generator=g).half().cuda()
    c = census.Census(ops, check_all=(height, width, n) == (1024, 1024, 1), plan=plan).install(monkeypatch)
    feats = sdxl_adapter(x)
    monkeypatch.undo()
    torch.cuda.synchronize()
    h, w = height // 16, width // 16
    assert [tuple(f.shape) for f in feats] == [(n, h, w, 320), (n, h, w, 640), (n, h // 2, w // 2, 1280),
                                               (n, h // 2, w // 2, 1280)]
    ops_seen = [r["op"] for r in c.rows.values()]
    assert {"conv3x3", "linear", "conv3x3_down"} <= set(ops_seen)
    flags = {(r["op"], f) for r in c.rows.values() for f in r["shape"].split()}
    assert ("conv3x3", "relu") in flags, "block1 must run with the ReLU epilogue"
    _finish(c, f"T2I-Adapter {height}x{width} n={n}")
