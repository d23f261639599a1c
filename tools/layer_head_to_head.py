"""BASELINE config 2 head-to-head for ONE IMAGHarmony cross-attention layer (SURVEY §8 row a1: C = 1280, 20 heads,
e = [B, 77+4, 2048]): the native processor on the sm_90a kernels vs the restated reference processor
(oracle.adapter_ref.IPAttnProcessorRef, pinned against ip_adapter/attention_processor.py:364-465) in torch-eager
fp16 on the same GPU (cuBLAS + torch SDPA) -- both timed as CUDA-graph replays so that host launch overhead does not
count, plus the reference's eager time.  Writes tools_out/layer_head_to_head.json.  Context, not a bench arm."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from imagharmony_b200.unet import Attention  # noqa: E402
from ip_adapter.attention_processor import IPAttnProcessor2_0  # noqa: E402
from oracle import adapter_ref as A  # noqa: E402
from oracle.unet_ref import Attention as RefAttention  # noqa: E402
from tools.microbench import timeit  # noqa: E402


def eager_time(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e-3


def main():
    C, H, D, L, NI = 1280, 20, 2048, 81, 4
    rows = []
    g = torch.Generator("cpu").manual_seed(0)
    attn = Attention(C, H, D)
    proc = IPAttnProcessor2_0(C, D, scale=1.0, num_tokens=NI, skip=False)
    for p in list(attn.parameters()) + list(proc.parameters()):
        p.data = torch.randn(p.shape, generator=g) * 0.02
    ra = RefAttention(C, H, D)
    ra.load_state_dict(attn.state_dict())
    rp = A.IPAttnProcessorRef(C, D, scale=1.0, num_tokens=NI, skip=False)
    rp.load_state_dict(proc.state_dict())
    attn, proc, ra, rp = attn.half().cuda(), proc.half().cuda(), ra.half().cuda(), rp.half().cuda()
    with torch.no_grad():
        for B in (2, 8, 16):
            for N in (256, 576, 1024):
                hid = (torch.randn(B, N, C, generator=g)).half().cuda()
                ehs = (torch.randn(B, L, D, generator=g)).half().cuda()
                flops = 2 * 2.0 * B * N * C * C + 4.0 * B * H * N * L * 64 + 2 * 2.0 * B * L * D * C * 2
                out_n = proc(attn, hid, encoder_hidden_states=ehs)            # also fills the K/V cache (hoisted work)
                out_r = rp(ra, hid, encoder_hidden_states=ehs)
                err = (out_n.float() - out_r.float()).abs().max().item()
                t_nat = timeit(lambda: proc(attn, hid, encoder_hidden_states=ehs))
                def cold():
                    proc._kv = None            # drop the cached K/V: the projections run again, as in the reference
                    return proc(attn, hid, encoder_hidden_states=ehs)
                t_nat_cold = timeit(cold)
                t_ref_graph = timeit(lambda: rp(ra, hid, encoder_hidden_states=ehs))
                t_ref_eager = eager_time(lambda: rp(ra, hid, encoder_hidden_states=ehs))
                rows.append({"unet_batch": B, "tokens": N, "max_abs_diff_vs_eager_fp16": err,
                             "native_us": t_nat * 1e6, "native_with_kv_projection_us": t_nat_cold * 1e6,
                             "reference_eager_graph_us": t_ref_graph * 1e6, "reference_eager_us": t_ref_eager * 1e6,
                             "speedup_vs_graph_replayed_reference": t_ref_graph / t_nat,
                             "native_tflops_incl_hoisted_flops": flops / t_nat / 1e12,
                             # FLOPs the per-step layer actually executes (to_q + decoupled attention + to_out; the K/V
                             # projections are hoisted out of the loop): what "fraction of tensor peak" must be quoted on
                             "native_tflops_executed": (2 * 2.0 * B * N * C * C + 4.0 * B * H * N * L * 64) / t_nat / 1e12})
                print(json.dumps(rows[-1]), flush=True)
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "tools_out", "layer_head_to_head.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
