"""Host-side algebra that the kernels rely on, checked in float64 on the CPU (no library needed)."""
import torch
import torch.nn.functional as F


def test_fold_layernorm_identity():
    """ops.fold_layernorm: LayerNorm(x) W^T + b == rstd(x) * (x Wc^T) + c with Wc = W gamma - rowmean(W gamma),
    c = W beta + b -- the centred weight makes the mean term vanish inside the GEMM (gemm.cu epilogue)."""
    from imagharmony_b200.ops import fold_layernorm
    g = torch.Generator().manual_seed(0)
    M, K, N = 37, 192, 64
    x = (torch.randn(M, K, generator=g) * 2 + 0.7).double()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half()
    b = torch.randn(N, generator=g).half()
    gamma = (1 + 0.3 * torch.randn(K, generator=g)).half()
    beta = (0.2 * torch.randn(K, generator=g)).half()
    w_c, c = fold_layernorm(w, b, gamma, beta)
    assert w_c.dtype == torch.float16 and c.dtype == torch.float16
    assert (w_c.double().sum(dim=1) == 0).all()                        # fp16 rows centred exactly
    mean = x.mean(dim=1, keepdim=True)
    rstd = torch.rsqrt(x.var(dim=1, unbiased=False, keepdim=True) + 1e-5)
    folded = rstd * (x @ w_c.double().t()) + c.double()
    ref = F.layer_norm(x, (K,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()
    # the only differences are the fp16 roundings of Wc and c
    assert (folded - ref).abs().max() < 5e-3, (folded - ref).abs().max()
    # and the statistics a producer GEMM hands over (sum, sum of squares per 64-column slab) rebuild mean / rstd
    slabs = x.reshape(M, K // 64, 64)
    s, q = slabs.sum(-1).sum(-1), (slabs * slabs).sum(-1).sum(-1)
    m2 = s / K
    r2 = torch.rsqrt((q / K - m2 * m2).clamp_min(0) + 1e-5)
    assert torch.allclose(m2, mean[:, 0]) and torch.allclose(r2, rstd[:, 0], rtol=1e-9)


def test_fold_rounding_keeps_rows_summing_to_zero():
    """The folded weight's fp16 rounding: every row sums to exactly zero (so mean(x) drops out of the GEMM at any
    |mean| / std), and the elementwise error stays that of round-to-nearest."""
    from imagharmony_b200.ops import _round_rows_zero_sum
    g = torch.Generator().manual_seed(1)
    for N, K, scale in [(1280, 1280, 1280 ** -0.5), (96, 320, 0.3), (40, 5120, 5120 ** -0.5 * 1e-3)]:
        w = torch.randn(N, K, generator=g, dtype=torch.float64) * scale
        w = w - w.mean(dim=1, keepdim=True)
        h = _round_rows_zero_sum(w)
        near = w.half()
        assert h.dtype == torch.float16 and (h.double().sum(dim=1) == 0).all()
        worst = (near.double() - w).abs().amax(dim=1)
        assert ((h.double() - w).abs().amax(dim=1) <= 2 * worst).all(), "a move larger than the row's rounding steps"
        rms = lambda t: (t.double() - w).pow(2).mean().sqrt().item()   # noqa: E731
        assert rms(h) <= 1.01 * rms(near), (rms(h), rms(near))
        assert (near.double().sum(dim=1) != 0).any()                   # round-to-nearest alone does not do it


def test_vae_folded_input_conv_matches_three_separate_ops():
    """vae.finalize: post_quant_conv (1x1) -> / scaling_factor -> conv_in (3x3, zero padding) as ONE patch-matrix product
    with a constant-one channel; exact at the image border, where a folded bias alone would be wrong."""
    from imagharmony_b200.config import TINY_VAE
    from imagharmony_b200.vae import AutoencoderKLDecoder
    torch.manual_seed(1)
    m = AutoencoderKLDecoder(TINY_VAE).double()
    m.decoder.conv_in.weight.data.normal_(0, 0.2)
    m.post_quant_conv.weight.data.normal_(0, 0.5)
    m.post_quant_conv.bias.data.normal_(0, 0.5)
    L, C0 = TINY_VAE.latent_channels, m.decoder.conv_in.weight.shape[0]
    # the same folding as AutoencoderKLDecoder.finalize, in float64
    wt = m.decoder.conv_in.weight.reshape(C0, L, 9)
    folded = torch.zeros(C0, L + 1, 9, dtype=torch.float64)
    folded[:, :L] = torch.einsum("omt,mc->oct", wt, m.post_quant_conv.weight.reshape(L, L)) / TINY_VAE.scaling_factor
    folded[:, L] = torch.einsum("omt,m->ot", wt, m.post_quant_conv.bias)
    z = torch.randn(2, L, 5, 7, dtype=torch.float64)
    z5 = torch.cat([z, torch.ones(2, 1, 5, 7, dtype=torch.float64)], dim=1)
    cols = F.unfold(z5, kernel_size=3, padding=1).transpose(1, 2)                       # [B, HW, (L+1)*9], k = c*9 + tap
    got = cols @ folded.reshape(C0, (L + 1) * 9).t() + m.decoder.conv_in.bias
    want = m.decoder.conv_in(m.post_quant_conv(z / TINY_VAE.scaling_factor))
    want = want.permute(0, 2, 3, 1).reshape(2, 35, C0)
    assert torch.allclose(got, want, atol=1e-10), (got - want).abs().max()
    # a plain folded bias (no ones channel) is wrong exactly at the border pixels
    naive = cols[..., :L * 9] @ folded[:, :L].reshape(C0, L * 9).t() + m.decoder.conv_in.bias + folded[:, L].sum(-1)
    err = (naive - want).abs().reshape(2, 5, 7, C0).amax(dim=(0, 3))
    assert err[1:-1, 1:-1].max() < 1e-10 and err[0].min() > 1e-6
