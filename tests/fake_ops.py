"""TEST-ONLY stand-ins for imagharmony_b200.ops implemented with plain PyTorch in fp32.  They let the CPU test suite
validate the *wiring* of the native UNet / processors / denoise loop (layouts, skip order, weight packing, K/V caching)
against the oracle without a GPU, and they are the per-call reference of the GPU census (tests/census.py), so they run
on whatever device their inputs live on.  Never imported by the product."""
import math

import torch
import torch.nn.functional as F

_count = [0]


def launch_count():
    return _count[0]


def launch_count_reset():
    _count[0] = 0


def fold_layernorm(w, bias, gamma, beta):
    w_g = w.double() * gamma.double()[None, :]
    w_c = (w_g - w_g.mean(dim=1, keepdim=True)).to(w.dtype).contiguous()
    c = w.double() @ beta.double()
    if bias is not None:
        c = c + bias.double()
    return w_c, c.to(w.dtype)


def _up(t):
    """fp32 compute for fp16 / fp32 operands; fp64 operands stay fp64 (the census' exact GEMM / conv references)."""
    return t if t.dtype == torch.float64 else t.float()


def linear(x, w, bias=None, *, residual=None, rowbias=None, rows_per_group=0, geglu=False, silu=False, gelu=False,
           out=None, tile_n=0, ln=None, stats_out=None, quick_gelu=False, alpha=1.0, relu=False):
    _count[0] += 1
    y = (_up(x) @ _up(w).t()) * alpha
    if ln is not None:
        st, eps = ln
        K = x.shape[1]
        tot = st.float().sum(dim=0)
        mean = tot[:, 0] / K
        var = (tot[:, 1] / K - mean * mean).clamp_min(0)
        y = torch.rsqrt(var + eps)[:, None] * y
    if bias is not None:
        y = y + bias.float()
    if geglu:
        a, g = y.chunk(2, dim=-1)
        y = a * F.gelu(g)
    if rowbias is not None:
        y = y + rowbias.float().repeat_interleave(rows_per_group, dim=0)
    if silu:
        y = F.silu(y)
    if gelu:
        y = F.gelu(y)
    if quick_gelu:
        y = y * torch.sigmoid(1.702 * y)
    if residual is not None:
        y = y + residual.float()
    if relu:                                # IH_EPI_RELU: after the residual
        y = torch.relu(y)
    y = y.to(x.dtype)
    if stats_out is not None:
        yf = y.float()
        n = yf.shape[1]
        pad = (-n) % 64
        yp = F.pad(yf, (0, pad)).reshape(yf.shape[0], -1, 64)
        stats_out.copy_(torch.stack([yp.sum(-1), (yp * yp).sum(-1)], dim=-1).transpose(0, 1))
    if out is not None:
        out.copy_(y)
        return out
    return y


def attention_small(q, k, v, B, H, Nq, Nk, dqk, dv, scale, out=None):
    _count[0] += 1
    qf = q.float().reshape(B, Nq, H, dqk).transpose(1, 2)
    kf = k.float().reshape(B, Nk, H, dqk).transpose(1, 2)
    vf = v.float().reshape(B, Nk, H, dv).transpose(1, 2)
    o = torch.softmax(qf @ kf.transpose(-1, -2) / scale, -1) @ vf
    return o.transpose(1, 2).reshape(B * Nq, H * dv).to(q.dtype)


def softmax_rows_masked_(x, valid_cols):
    _count[0] += 1
    y = torch.zeros_like(x, dtype=torch.float32)
    y[:, :valid_cols] = torch.softmax(x[:, :valid_cols].float(), dim=-1)
    x.copy_(y.to(x.dtype))
    return x


def add_bcast(a, b, out=None):
    _count[0] += 1
    return (a.reshape(-1, b.numel()) + b.reshape(1, -1)).reshape(a.shape)


def mean_tokens(x, out=None):
    _count[0] += 1
    return x.mean(dim=1)


def pack_conv3x3_weight(w):
    Cout, Cin, _, _ = w.shape
    return w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()


def conv3x3(x, w_packed, bias=None, *, rowbias=None, residual=None, stride=1, out=None, tile_n=0, alpha=1.0, shortcut=None,
            relu=False):
    _count[0] += 1
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    sc_term = None
    if shortcut is not None:
        src = shortcut[0] if shortcut[1] is None else torch.cat([shortcut[0], shortcut[1]], dim=-1)
        sc_term = _up(src) @ _up(w_packed[:, 9 * Cin:]).t()
        w_packed = w_packed[:, : 9 * Cin]
    w = _up(w_packed.reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2))
    y = F.conv2d(_up(x).permute(0, 3, 1, 2), w, None, stride=stride, padding=1).permute(0, 2, 3, 1) * alpha
    if bias is not None:
        y = y + bias.float()
    if rowbias is not None:
        y = y + rowbias.float()[:, None, None, :]
    if residual is not None:
        y = y + residual.float()
    if sc_term is not None:
        y = y + sc_term
    if relu:                                # IH_EPI_RELU: after the residual
        y = torch.relu(y)
    return y.to(x.dtype).contiguous()


def attention(q, k, v, B, H, Nq, Nk, *, n_ip=0, ip_scale=1.0, out=None, kv_split=True):
    _count[0] += 1
    C = H * 64
    qf = q.float().reshape(B, Nq, H, 64).transpose(1, 2)
    kf = k.float().reshape(B, Nk, H, 64).transpose(1, 2)
    vf = v.float().reshape(B, Nk, H, 64).transpose(1, 2)
    nt = Nk - n_ip
    o = torch.softmax(qf @ kf[:, :, :nt].transpose(-1, -2) / 8.0, -1) @ vf[:, :, :nt]
    if n_ip > 0:
        o = o + ip_scale * (torch.softmax(qf @ kf[:, :, nt:].transpose(-1, -2) / 8.0, -1) @ vf[:, :, nt:])
    return o.transpose(1, 2).reshape(B * Nq, C).to(q.dtype)


def groupnorm(x0, gamma, beta, *, x1=None, groups=32, eps=1e-5, silu=False, out=None, ws=None):
    _count[0] += 2
    x = x0 if x1 is None else torch.cat([x0, x1], dim=-1)
    y = F.group_norm(x.float().permute(0, 3, 1, 2), groups, gamma.float(), beta.float(), eps)
    if silu:
        y = F.silu(y)
    return y.permute(0, 2, 3, 1).to(x0.dtype).contiguous()


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    _count[0] += 1
    return F.layer_norm(x.float(), (x.shape[-1],), gamma.float(), beta.float(), eps).to(x.dtype)


def linear_small(x, w, bias=None, *, act_in=False, act_out=False, addend=None, out_scale=1.0, out=None):
    _count[0] += 1
    xi = F.silu(x.float()) if act_in else x.float()
    y = xi @ w.float().t()
    if bias is not None:
        y = y + bias.float()
    if act_out:
        y = F.silu(y)
    y = y * out_scale
    if addend is not None:
        y = y + addend.float()
    y = y.to(x.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def sinusoid(t, dim, n, *, step=None, out=None):
    _count[0] += 1
    half = dim // 2
    tv = t[step.long()].expand(n) if step is not None else t[:n]
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    a = tv.float().reshape(-1, 1) * f.reshape(1, -1)
    return torch.cat([a.cos(), a.sin()], -1).to(torch.float32 if FP32 else torch.float16)


FP32 = True


def upsample2x(x, out=None):
    _count[0] += 1
    return F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1).contiguous()


def concat_channels(x0, x1, out=None):
    _count[0] += 1
    return torch.cat([x0, x1], dim=-1)


def euler_cfg_step(noise_pred, latents, model_in, sigmas, step, guidance):
    _count[0] += 2
    i = int(step.item())
    s, sn = float(sigmas[i]), float(sigmas[i + 1])
    u, c = noise_pred.chunk(2)
    eps = u + guidance * (c - u)
    x = latents.float()
    x0 = x - (s * eps.float()).to(eps.dtype).float()
    xn = (x + (x - x0) / s * (sn - s)).to(latents.dtype)
    latents.copy_(xn)
    mi = (xn.float() / (sn * sn + 1) ** 0.5).to(model_in.dtype)
    model_in.copy_(torch.cat([mi, mi]))
    step += 1


def workspace_generation():
    return 0


def prefetch_next(w):
    return None


def euler_step(noise_pred, latents, model_in, sigmas, step, guidance, *, use_cfg=True, guidance_rescale=0.0):
    if use_cfg and not guidance_rescale:
        return euler_cfg_step(noise_pred, latents, model_in, sigmas, step, guidance)
    _count[0] += 2
    i = int(step.item())
    s, sn = float(sigmas[i]), float(sigmas[i + 1])
    if use_cfg:
        u, c = noise_pred.chunk(2)
        eps = u + guidance * (c - u)
        dims = list(range(1, eps.dim()))
        resc = eps * (c.std(dim=dims, keepdim=True) / eps.std(dim=dims, keepdim=True))
        eps = guidance_rescale * resc + (1 - guidance_rescale) * eps
    else:
        eps = noise_pred
    x = latents.float()
    x0 = x - (s * eps.float()).to(eps.dtype).float()
    xn = (x + (x - x0) / s * (sn - s)).to(latents.dtype)
    latents.copy_(xn)
    mi = (xn.float() / (sn * sn + 1) ** 0.5).to(model_in.dtype)
    model_in.copy_(torch.cat([mi, mi]) if use_cfg else mi)
    step += 1


def scale_model_input(latents, model_in, sigmas, step, duplicate=True):
    _count[0] += 1
    s = float(sigmas[int(step.item())])
    mi = (latents.float() / (s * s + 1) ** 0.5).to(model_in.dtype)
    model_in.copy_(torch.cat([mi, mi]) if duplicate else mi)


def im2col3x3_nchw(x_nchw, kpad=64, out=None):
    _count[0] += 1
    B, C, H, W = x_nchw.shape
    cols = F.unfold(x_nchw.float(), kernel_size=3, padding=1)            # [B, C*9, H*W], k = c*9 + ky*3 + kx
    a = cols.transpose(1, 2).reshape(B * H * W, C * 9)
    return F.pad(a, (0, kpad - C * 9)).to(x_nchw.dtype)


def nhwc_to_nchw(x, C, out=None):
    _count[0] += 1
    return x[..., :C].permute(0, 3, 1, 2).contiguous()


def attention_generic(q, k, v, B, H, Nq, Nk, dqk, dv, scale, causal=False, out=None):
    _count[0] += 1
    qh = q[:, :H * dqk].float().reshape(B, Nq, H, dqk).permute(0, 2, 1, 3)
    kh = k[:, :H * dqk].float().reshape(B, Nk, H, dqk).permute(0, 2, 1, 3)
    vh = v[:, :H * dv].float().reshape(B, Nk, H, dv).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * scale
    if causal:
        mask = torch.ones(Nq, Nk, dtype=torch.bool, device=q.device).tril(Nk - Nq)
        s = s.masked_fill(~mask, float("-inf"))
    o = (s.softmax(-1) @ vh).permute(0, 2, 1, 3).reshape(B * Nq, H * dv).to(q.dtype)
    if out is not None:
        out.copy_(o)
        return out
    return o


def embed_tokens(ids, tok_emb, pos_emb, out=None):
    _count[0] += 1
    B, T = ids.shape
    return (tok_emb[ids.long()] + pos_emb[:T][None]).reshape(B * T, -1)


def resize_patchify(img, size, patch, kpad, mean, std, out=None):
    _count[0] += 1
    from oracle.clip_ref import resize_patchify_ref
    return resize_patchify_ref(img.float(), size, patch, kpad, mean, std).to(img.dtype)
