"""ORACLE (test infrastructure only) for Euler Ancestral: a CPU / any-device restatement of what [3P]
diffusers==0.30.0 `EulerAncestralDiscreteScheduler` (requirements.txt:25; not vendored) does with the SDXL-base
scheduler_config, and of the `randn_tensor` draws its `step` makes.  **Parity unpinned**, like the other [3P]
restatements: diffusers is not installable here; it follows the diffusers 0.30.0 sources as published (SURVEY A.6,
C.28-C.31).  Written independently of imagharmony_b200/scheduler.py:

* `randn_tensor_ref`: diffusers.utils.torch_utils.randn_tensor (generator device, list of generators, None);
* `EulerAncestralRef`: the stateful scheduler with diffusers' tensor expressions and 0-dim fp32 CPU sigmas, so the
  dtypes and devices of the tensors it is given decide the rounding points (fp32 oracle, fp16 CUDA for the kernel);
* `euler_a_denoise_loop`: the loop of custom_pipelines.py:325-363 with this scheduler, optionally image-to-image
  (`begin`) and with the 4-channel inpainting blend (`blend`);
* `euler_a_step_ref`: one guided step on given tensors and noise -- the restatement the kernel is tested against;
* `masked_image_draw_ref`: the posterior draw of the masked-image encode of the inpainting pipeline (C.31).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from img2img_ref import add_noise_ref
from oracle.scheduler_ref import euler_tables, rescale_noise_cfg


def randn_tensor_ref(shape, generator, device, dtype):
    device = torch.device(device)
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        rand_device = generator[0].device
        parts = [torch.randn((1,) + tuple(shape[1:]), generator=generator[i], device=rand_device, dtype=dtype)
                 for i in range(shape[0])]
        return torch.cat(parts, dim=0).to(device)
    rand_device = generator.device if generator is not None else device
    return torch.randn(tuple(shape), generator=generator, device=rand_device, dtype=dtype).to(device)


class EulerAncestralRef:
    def __init__(self, num_inference_steps: int):
        ts, sig, ins = euler_tables(num_inference_steps)       # the tables are Euler's (SURVEY A.6)
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.from_numpy(sig).to("cpu")
        self.init_noise_sigma = ins
        self.step_index = 0

    def scale_model_input(self, sample):
        sigma = self.sigmas[self.step_index]
        return sample / ((sigma**2 + 1) ** 0.5)

    def step(self, model_output, sample, generator=None, noise=None, noise_dtype=None):
        """`noise` given: used instead of a draw (the kernel test); else drawn like diffusers, in `noise_dtype`
        (the pipeline's fp16 when the oracle computes in fp32) and used in the model output's dtype."""
        sigma = self.sigmas[self.step_index]
        sample = sample.to(torch.float32)
        pred_original_sample = sample - sigma * model_output
        sigma_from = self.sigmas[self.step_index]
        sigma_to = self.sigmas[self.step_index + 1]
        sigma_up = (sigma_to**2 * (sigma_from**2 - sigma_to**2) / sigma_from**2) ** 0.5
        sigma_down = (sigma_to**2 - sigma_up**2) ** 0.5
        derivative = (sample - pred_original_sample) / sigma
        dt = sigma_down - sigma
        prev_sample = sample + derivative * dt
        if noise is None:
            noise = randn_tensor_ref(model_output.shape, generator, model_output.device,
                                     noise_dtype or model_output.dtype)
        prev_sample = prev_sample + noise.to(model_output.device, model_output.dtype) * sigma_up
        self.step_index += 1
        return prev_sample.to(model_output.dtype)


def _guided(noise_pred, guidance_scale, guidance_rescale, cfg):
    if not cfg:
        return noise_pred
    u, c = noise_pred.chunk(2)
    eps = u + guidance_scale * (c - u)
    if guidance_rescale > 0.0:
        eps = rescale_noise_cfg(eps, c, guidance_rescale)
    return eps


@torch.no_grad()
def euler_a_denoise_loop(unet_fn: Callable, latents, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled, time_ids,
                         num_inference_steps: int, generator=None, guidance_scale: float = 5.0,
                         set_scale: Optional[Callable[[float], None]] = None, conditioning_scale: float = 1.0,
                         control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                         guidance_rescale: float = 0.0, denoising_end: Optional[float] = None,
                         callback: Optional[Callable] = None, callback_steps: int = 1, begin: int = 0, blend=None,
                         noise_dtype=torch.float16) -> torch.Tensor:
    """custom_pipelines.py:296-363 with Euler Ancestral over timesteps[begin:] (image-to-image: `latents` already carry
    the noise of sigma[begin]).  `blend` = (image_latents, noise, mask): after every step the 4-channel inpainting blend
    with the image latents re-noised to the next sigma, the clean ones after the last step of the loop."""
    sched = EulerAncestralRef(num_inference_steps)
    sched.step_index = begin
    ts = sched.timesteps[begin:].tolist()
    if denoising_end is not None and isinstance(denoising_end, float) and 0 < denoising_end < 1:
        cutoff = int(round(1000 - denoising_end * 1000))
        ts = ts[:sum(1 for t in ts if t >= cutoff)]
    n_loop = len(ts)
    cfg = guidance_scale > 1.0
    if cfg:
        ehs = torch.cat([neg_prompt_embeds, prompt_embeds], dim=0)
        text_embeds = torch.cat([neg_pooled, pooled], dim=0)
        tids = torch.cat([time_ids, time_ids], dim=0)
    else:
        ehs, text_embeds, tids = prompt_embeds, pooled, time_ids
    for i in range(n_loop):
        if set_scale is not None:
            off = (i / n_loop < control_guidance_start) or ((i + 1) / n_loop > control_guidance_end)
            set_scale(0.0 if off else conditioning_scale)
        x2 = torch.cat([latents] * 2) if cfg else latents
        x2 = sched.scale_model_input(x2).to(latents.dtype)
        noise_pred = unet_fn(x2, float(ts[i]), ehs, text_embeds, tids)
        eps = _guided(noise_pred, guidance_scale, guidance_rescale, cfg)
        latents = sched.step(eps, latents, generator, noise_dtype=noise_dtype)
        if blend is not None:
            image_latents, noise, mask = blend
            proper = image_latents
            if i < n_loop - 1:
                proper = add_noise_ref(image_latents, noise, float(sched.sigmas[sched.step_index]))
            latents = (1 - mask) * proper + mask * latents
        if callback is not None and i % callback_steps == 0:
            callback(i, float(ts[i]), latents)
    return latents


def euler_a_step_ref(noise_pred, latents, num_inference_steps: int, i: int, guidance: float, step_noise,
                     use_cfg: bool = True, guidance_rescale: float = 0.0, blend=None, blend_end: Optional[int] = None):
    """Step i of the schedule on the given tensors (any device) with the given noise -> (latents, next model input);
    `blend` = (image_latents, noise, mask) with the loop ending at schedule index `blend_end`."""
    sched = EulerAncestralRef(num_inference_steps)
    sched.step_index = i
    x = sched.step(_guided(noise_pred, guidance, guidance_rescale, use_cfg), latents, noise=step_noise)
    if blend is not None:
        image_latents, noise, mask = blend
        proper = image_latents
        if i + 1 < blend_end:
            proper = add_noise_ref(image_latents, noise, float(sched.sigmas[i + 1]))
        x = (1 - mask) * proper + mask * x
    mi = sched.scale_model_input(x)
    return x, (torch.cat([mi, mi]) if use_cfg else mi)


def masked_image_draw_ref(n_masked: int, latent_shape, generator, dtype=torch.float32) -> None:
    """`_encode_vae_image(masked_image, generator)`: the posterior eps of the masked images, drawn and unused with the
    4-channel UNet (image i with generator[i] for a list)."""
    if isinstance(generator, list):
        for g in generator[:n_masked]:
            torch.randn((1,) + tuple(latent_shape), generator=g, device=g.device, dtype=dtype)
    else:
        torch.randn((n_masked,) + tuple(latent_shape), generator=generator, dtype=dtype)
