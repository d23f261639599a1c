"""TEST-ONLY restatement of [3P] diffusers 0.30.0 MultiControlNetModel.forward and of StableDiffusionXLControlNetPipeline's
loop with a MultiControlNetModel (the alignment of scales and guidance windows, controlnet_keep as one list per net,
cond_scale = scale_k * keep_k, inactive nets run at scale 0), fp32 or fp16, on the ControlNetRef / UNetResidualRef of
tests/controlnet_ref.py."""
import torch


def multi_forward_ref(controlnets, sample, timestep, ehs, images, scales, text_embeds, time_ids, guess_mode=False):
    """MultiControlNetModel.forward: each net's scaled residuals (ControlNetRef returns them scaled), added in net order;
    -> (down list, mid)."""
    down = mid = None
    for i, (cn, image, scale) in enumerate(zip(controlnets, images, scales)):
        d, m = cn(sample, timestep, ehs, image, scale, text_embeds, time_ids, guess_mode=guess_mode)
        if i == 0:
            down, mid = d, m
        else:
            down = [a + b for a, b in zip(down, d)]
            mid = mid + m
    return down, mid


def align_ref(n_nets, scale, start, end):
    """diffusers' alignment for a MultiControlNetModel -> (scales, starts, ends), one entry per net."""
    if not isinstance(start, list) and isinstance(end, list):
        start = len(end) * [start]
    elif not isinstance(end, list) and isinstance(start, list):
        end = len(start) * [end]
    elif not isinstance(start, list) and not isinstance(end, list):
        start, end = n_nets * [start], n_nets * [end]
    if isinstance(scale, float):
        scale = [scale] * n_nets
    return scale, start, end


@torch.no_grad()
def multi_controlnet_denoise_loop(unet, controlnets, latents, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled,
                                  time_ids, images, num_inference_steps, guidance_scale=5.0, conditioning_scale=1.0,
                                  guess_mode=False, control_guidance_start=0.0, control_guidance_end=1.0,
                                  scheduler="euler", generator=None):
    """The pipeline loop over `controlnets` (one image per net); the step is oracle.scheduler_ref's Euler step or, with
    scheduler="euler_a", tests/euler_a_ref.py's Euler Ancestral step with fp16 step noise from `generator`."""
    from euler_a_ref import EulerAncestralRef
    from oracle.scheduler_ref import euler_tables
    scales, starts, ends = align_ref(len(controlnets), conditioning_scale, control_guidance_start,
                                     control_guidance_end)
    timesteps, sigmas, _ = euler_tables(num_inference_steps)
    anc = EulerAncestralRef(num_inference_steps) if scheduler == "euler_a" else None
    cfg = guidance_scale > 1.0
    T = num_inference_steps
    ehs = torch.cat([neg_prompt_embeds, prompt_embeds]) if cfg else prompt_embeds
    te = torch.cat([neg_pooled, pooled]) if cfg else pooled
    tids = torch.cat([time_ids, time_ids]) if cfg else time_ids
    imgs = [torch.cat([im] * 2) if (cfg and not guess_mode) else im for im in images]
    for i in range(T):
        keeps = [1.0 - float(i / T < s or (i + 1) / T > e) for s, e in zip(starts, ends)]
        cond_scale = [c * k for c, k in zip(scales, keeps)]
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])
        x2 = torch.cat([latents] * 2) if cfg else latents
        x2 = x2 / ((sigma ** 2 + 1) ** 0.5)
        if guess_mode and cfg:
            n = latents.shape[0]
            down, mid = multi_forward_ref(controlnets, x2[n:], float(timesteps[i]), prompt_embeds, imgs, cond_scale,
                                          pooled, time_ids, guess_mode=True)
            down = [torch.cat([torch.zeros_like(d), d]) for d in down]
            mid = torch.cat([torch.zeros_like(mid), mid])
        else:
            down, mid = multi_forward_ref(controlnets, x2, float(timesteps[i]), ehs, imgs, cond_scale, te, tids,
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
