"""The persistent warp-specialised self-attention kernel (multi-block path, Nk > 128) against the two-CTA-per-SM kernel
it replaced there (ih_attention_set_kernel(1)) and the fp32 reference.  Rows processed whole evaluate the same
arithmetic in both kernels, so with the KV split withheld the outputs must be bit-identical."""
import pytest
import torch

pytestmark = pytest.mark.gpu

RTOL = ATOL = 1e-3


@pytest.fixture(scope="module")
def lib():
    from imagharmony_b200 import _lib
    lib = _lib.load()
    yield lib
    lib.ih_attention_set_kernel(0)
    lib.ih_attention_set_split_policy(0)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def sdpa_ref(q, k, v, B, H, Nq, Nk):
    qf = q.float().reshape(B, Nq, H, 64).transpose(1, 2)
    kf = k.float().reshape(B, Nk, H, 64).transpose(1, 2)
    vf = v.float().reshape(B, Nk, H, 64).transpose(1, 2)
    o = (qf @ kf.transpose(-1, -2) / 8.0).softmax(-1) @ vf
    return o.transpose(1, 2).reshape(B * Nq, H * 64)


def inputs(B, H, Nq, Nk, fused, qscale=1.0):
    C = H * 64
    if fused:   # strided views of one q|k|v projection output, row stride 3C (Nq == Nk) or two such buffers
        a = rnd(B * Nq, 3 * C, scale=qscale)
        b = a if Nq == Nk else rnd(B * Nk, 3 * C, seed=1)
        return a[:, :C], b[:, C:2 * C], b[:, 2 * C:]
    return rnd(B * Nq, C, scale=qscale), rnd(B * Nk, C, seed=1), rnd(B * Nk, C, seed=2)


def both(lib, ops, q, k, v, B, H, Nq, Nk, kv_split):
    outs = []
    for kern in (0, 1):
        lib.ih_attention_set_kernel(kern)
        try:
            outs.append(ops.attention(q, k, v, B, H, Nq, Nk, kv_split=kv_split))
        finally:
            lib.ih_attention_set_kernel(0)
    return outs


SHAPES = [(2, 10, 4096, 4096), (2, 20, 1024, 1024), (2, 20, 256, 256), (2, 5, 576, 576), (1, 2, 100, 300),
          (1, 3, 2000, 1500)]


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_new_kernel_bit_identical_to_old(lib, B, H, Nq, Nk, fused):
    from imagharmony_b200 import ops
    q, k, v = inputs(B, H, Nq, Nk, fused)
    new, old = both(lib, ops, q, k, v, B, H, Nq, Nk, kv_split=False)
    assert torch.equal(new, old), f"max |diff| {(new.float() - old.float()).abs().max().item():.3e}"
    torch.testing.assert_close(new.float(), sdpa_ref(q, k, v, B, H, Nq, Nk), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("B,H,Nq,Nk,qscale", [(2, 20, 1024, 1024, 1.0), (2, 10, 4096, 4096, 1.0),
                                               (2, 5, 576, 576, 3.0), (1, 3, 2000, 1500, 2.0)])
def test_split_path(lib, B, H, Nq, Nk, qscale, policy):
    from imagharmony_b200 import ops
    q, k, v = inputs(B, H, Nq, Nk, True, qscale)
    lib.ih_attention_set_split_policy(policy)
    try:
        if policy == 1:
            assert lib.ih_attention_workspace_bytes(B, H, Nq, Nk, 0) > 0, "shape does not exercise the split path"
        split = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=True)
        again = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=True)
        whole = ops.attention(q, k, v, B, H, Nq, Nk, kv_split=False)
    finally:
        lib.ih_attention_set_split_policy(0)
    ref = sdpa_ref(q, k, v, B, H, Nq, Nk)
    torch.testing.assert_close(split.float(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(whole.float(), ref, rtol=RTOL, atol=ATOL)
    assert torch.equal(split, again), "KV-split attention must be run-to-run deterministic"


def test_graph_replay_matches_eager(lib):
    from imagharmony_b200 import ops
    B, H, N = 2, 20, 1024
    q, k, v = inputs(B, H, N, N, True)
    out = torch.empty(B * N, H * 64, dtype=torch.float16, device="cuda")
    eager = ops.attention(q, k, v, B, H, N, N).clone()     # also creates the split workspace before capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        ops.attention(q, k, v, B, H, N, N, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


def _tiny_engine():
    from imagharmony_b200.config import TINY as cfg
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle.unet_ref import UNetRef
    with torch.device("meta"):
        shapes = shapes_of(UNetRef(cfg))
    native = UNet2DConditionModel.from_state_dict(cfg, random_state_dict(shapes, 0), device="cuda:0")
    procs = torch.nn.ModuleList(native.attn_processors.values())
    procs.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(procs), 1).items()})
    native.finalize()
    return cfg, native


def test_engine_batch_growth_bit_identical(lib):
    from imagharmony_b200.denoise import DenoiseEngine
    from oracle.scheduler_ref import euler_tables, prepare_latents
    cfg, native = _tiny_engine()
    T, lat = 2, 32
    _, _, ins = euler_tables(T)
    L = 77 + cfg.num_ip_tokens

    def args(n):
        g = torch.Generator("cpu").manual_seed(3)
        latents = prepare_latents(n, 4, lat, lat, list(range(42, 42 + n)), ins)
        pos = torch.randn(n, L, cfg.cross_attention_dim, generator=g).half()
        neg = torch.randn(n, L, cfg.cross_attention_dim, generator=g).half()
        pp = torch.randn(n, cfg.pooled_embed_dim, generator=g).half()
        npool = torch.randn(n, cfg.pooled_embed_dim, generator=g).half()
        tid = torch.tensor([[256.0, 256.0, 0, 0, 256.0, 256.0]] * n)
        return latents, pos, neg, pp, npool, tid, T

    eng = DenoiseEngine(native, use_cuda_graph=True)
    seq = [eng.run(*args(n), guidance_scale=5.0).clone() for n in (1, 4, 1)]
    for n, got in zip((1, 4, 1), seq):
        fresh = DenoiseEngine(native, use_cuda_graph=True).run(*args(n), guidance_scale=5.0)
        assert torch.equal(got, fresh), f"batch {n}"
    assert torch.equal(seq[0], seq[2])
