"""TEST-ONLY restatement of [3P] diffusers 0.30.0 ControlNetModel, of UNet2DConditionModel's
down_block_additional_residuals / mid_block_additional_residual, and of StableDiffusionXLControlNetPipeline's loop
(SURVEY appendix A.7), fp32 on the CPU, built on the oracle's UNet blocks (oracle/unet_ref.py).  It keeps diffusers'
form: ControlNetRef.forward returns the SCALED residuals, the UNet takes them as keyword arguments."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.unet_ref import DownBlock, MidBlock, TimestepEmbedding, UNetRef, sinusoidal_embedding


class ConditioningEmbeddingRef(nn.Module):
    def __init__(self, out_ch, cond_ch, widths):
        super().__init__()
        self.conv_in = nn.Conv2d(cond_ch, widths[0], 3, padding=1)
        blocks = []
        for c, c2 in zip(widths[:-1], widths[1:]):
            blocks.append(nn.Conv2d(c, c, 3, padding=1))
            blocks.append(nn.Conv2d(c, c2, 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        self.conv_out = nn.Conv2d(widths[-1], out_ch, 3, padding=1)

    def forward(self, x):
        x = F.silu(self.conv_in(x))
        for b in self.blocks:
            x = F.silu(b(x))
        return self.conv_out(x)


class ControlNetRef(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        boc, tl = cfg.block_out_channels, cfg.transformer_layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], cfg.time_embed_dim)
        self.add_embedding = TimestepEmbedding(cfg.add_embed_in, cfg.time_embed_dim)
        self.controlnet_cond_embedding = ConditioningEmbeddingRef(boc[0], cfg.conditioning_channels,
                                                                  cfg.conditioning_embedding_out_channels)
        downs, zc = [], [nn.Conv2d(boc[0], boc[0], 1)]
        ch = boc[0]
        for i, co in enumerate(boc):
            last = i == len(boc) - 1
            downs.append(DownBlock(cfg, ch, co, tl[i], add_down=not last))
            zc += [nn.Conv2d(co, co, 1) for _ in range(cfg.layers_per_block + (0 if last else 1))]
            ch = co
        self.down_blocks = nn.ModuleList(downs)
        self.controlnet_down_blocks = nn.ModuleList(zc)
        self.controlnet_mid_block = nn.Conv2d(boc[-1], boc[-1], 1)
        self.mid_block = MidBlock(cfg, boc[-1], tl[-1])

    attn_processors = UNetRef.attn_processors
    set_attn_processor = UNetRef.set_attn_processor

    def forward(self, sample, timestep, ehs, controlnet_cond, conditioning_scale, text_embeds, time_ids,
                guess_mode=False):
        cfg = self.config
        b = sample.shape[0]
        t = torch.full((b,), float(timestep), dtype=torch.float32, device=sample.device)
        emb = self.time_embedding(sinusoidal_embedding(t, cfg.block_out_channels[0]).to(sample.dtype))
        tid = sinusoidal_embedding(time_ids.reshape(-1).to(sample.device), cfg.addition_time_embed_dim).reshape(b, -1)
        emb = emb + self.add_embedding(torch.cat([text_embeds, tid.to(text_embeds.dtype)], dim=-1).to(sample.dtype))
        if cfg.controlnet_conditioning_channel_order == "bgr":
            controlnet_cond = torch.flip(controlnet_cond, dims=[1])
        x = self.conv_in(sample) + self.controlnet_cond_embedding(controlnet_cond)
        skips = [x]
        for blk in self.down_blocks:
            x = blk(x, emb, ehs, skips)
        x = self.mid_block(x, emb, ehs)
        down = [z(s) for z, s in zip(self.controlnet_down_blocks, skips)]
        mid = self.controlnet_mid_block(x)
        if guess_mode:
            scales = torch.logspace(-1, 0, len(down) + 1) * conditioning_scale
            down = [d * s for d, s in zip(down, scales)]
            mid = mid * scales[-1]
        else:
            down = [d * conditioning_scale for d in down]
            mid = mid * conditioning_scale
        return down, mid

    def raw(self, *a, **k):
        """The unscaled zero-conv outputs (conditioning_scale 1, no guess mode)."""
        down, mid = self.forward(*a, **k)
        return down + [mid]


class UNetResidualRef(UNetRef):
    """UNetRef whose forward also takes diffusers' down_block_additional_residuals / mid_block_additional_residual.
    UNetRef.forward itself runs; for one call the mid block's output gets the mid residual and, as the first up block
    starts, the complete skip list gets the down residuals (diffusers adds them after the down path)."""

    def forward(self, sample, timestep, encoder_hidden_states, text_embeds, time_ids,
                down_block_additional_residuals=None, mid_block_additional_residual=None):
        args = (sample, timestep, encoder_hidden_states, text_embeds, time_ids)
        if down_block_additional_residuals is None and mid_block_additional_residual is None:
            return super().forward(*args)
        mid_fwd, up_fwd = self.mid_block.forward, self.up_blocks[0].forward

        def mid_plus(*a):
            x = mid_fwd(*a)
            return x if mid_block_additional_residual is None else x + mid_block_additional_residual

        def up_first(x, emb, ehs, skips):
            if down_block_additional_residuals is not None:
                assert len(skips) == len(down_block_additional_residuals)
                skips[:] = [s + r for s, r in zip(skips, down_block_additional_residuals)]
            return up_fwd(x, emb, ehs, skips)
        self.mid_block.forward, self.up_blocks[0].forward = mid_plus, up_first
        try:
            return super().forward(*args)
        finally:
            del self.mid_block.forward, self.up_blocks[0].forward


@torch.no_grad()
def controlnet_denoise_loop(unet, controlnet, latents, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled, time_ids,
                            image, num_inference_steps, guidance_scale=5.0, conditioning_scale=1.0, guess_mode=False,
                            control_guidance_start=0.0, control_guidance_end=1.0, scheduler="euler", generator=None):
    """[3P] StableDiffusionXLControlNetPipeline's loop with the Euler step of oracle.scheduler_ref.denoise_loop, or
    with scheduler="euler_a" the Euler Ancestral step of tests/euler_a_ref.py (step noise drawn from `generator` in
    fp16, one draw per step, as diffusers draws it)."""
    from euler_a_ref import EulerAncestralRef
    from oracle.scheduler_ref import euler_tables
    timesteps, sigmas, _ = euler_tables(num_inference_steps)
    anc = EulerAncestralRef(num_inference_steps) if scheduler == "euler_a" else None
    cfg = guess_cfg = guidance_scale > 1.0
    T = num_inference_steps
    ehs = torch.cat([neg_prompt_embeds, prompt_embeds]) if cfg else prompt_embeds
    te = torch.cat([neg_pooled, pooled]) if cfg else pooled
    tids = torch.cat([time_ids, time_ids]) if cfg else time_ids
    img = torch.cat([image] * 2) if (cfg and not guess_mode) else image
    for i in range(T):
        keep = 1.0 - float(i / T < control_guidance_start or (i + 1) / T > control_guidance_end)
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])
        x2 = torch.cat([latents] * 2) if cfg else latents
        x2 = x2 / ((sigma ** 2 + 1) ** 0.5)
        if guess_mode and guess_cfg:
            n = latents.shape[0]
            down, mid = controlnet(x2[n:], float(timesteps[i]), prompt_embeds, img, conditioning_scale * keep,
                                   pooled, time_ids, guess_mode=True)
            down = [torch.cat([torch.zeros_like(d), d]) for d in down]
            mid = torch.cat([torch.zeros_like(mid), mid])
        else:
            down, mid = controlnet(x2, float(timesteps[i]), ehs, img, conditioning_scale * keep, te, tids,
                                   guess_mode=guess_mode)
        noise = unet(x2, float(timesteps[i]), ehs, te, tids, down_block_additional_residuals=down,
                     mid_block_additional_residual=mid)
        if cfg:
            u, c = noise.chunk(2)
            eps = u + guidance_scale * (c - u)
        else:
            eps = noise
        if anc is not None:
            latents = anc.step(eps, latents, generator, noise_dtype=torch.float16)
            continue
        x0 = latents - sigma * eps
        latents = latents + (latents - x0) / sigma * (sigma_next - sigma)
    return latents
