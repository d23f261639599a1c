"""ORACLE (test infrastructure only) for inpainting with the 4-channel SDXL-base UNet: CPU restatements of what
[3P] diffusers==0.30.0 `StableDiffusionXLInpaintPipeline` (requirements.txt:25; not vendored) adds on top of
image-to-image.  **Parity unpinned**, like the other [3P] restatements: diffusers is not installable here and the
reference holds no golden vector for these; they follow the diffusers 0.30.0 sources as published (SURVEY C.19-C.21).

* `preprocess_mask_ref`: `VaeImageProcessor(do_normalize=False, do_binarize=True, do_convert_grayscale=True)`;
* `mask_latents_ref`: `prepare_mask_latents` -- nearest `interpolate` to the latent size, fp16, `repeat` to the batch;
* `prepare_inpaint_latents`: `prepare_latents(return_image_latents=True)` -- image latents, noise, start latents and the
  RNG order (posterior eps first; with a list of generators only the images encode, with generator[i]);
* `inpaint_denoise_loop`: the loop over timesteps[t_start:] with the 4-channel blend after every `scheduler.step`;
* `inpaint_step_ref`: the rounding points of ih_euler_inpaint_step as torch ops on any device.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from img2img_ref import _randn, add_noise_ref, img2img_timesteps, posterior_sample_ref
from oracle.scheduler_ref import euler_tables, rescale_noise_cfg


def preprocess_mask_ref(mask, height: int, width: int) -> torch.Tensor:
    """PIL: convert("L"), resize((width, height), LANCZOS), / 255 -> [B,1,H,W]; tensor: grayscale dim inserted, nearest
    interpolate; then binarize (< 0.5 -> 0, >= 0.5 -> 1)."""
    from PIL import Image
    if isinstance(mask, torch.Tensor):
        x = mask.float()
        if x.ndim == 3:
            x = x.unsqueeze(1)
        elif x.ndim == 2:
            x = torch.stack([x], dim=0).unsqueeze(1)
        x = F.interpolate(x, size=(height, width))
    else:
        masks = mask if isinstance(mask, list) else [mask]
        masks = [m.convert("L").resize((width, height), resample=Image.LANCZOS) for m in masks]
        arr = np.stack([np.array(m).astype(np.float32) / 255.0 for m in masks])[..., None]
        x = torch.from_numpy(arr).permute(0, 3, 1, 2)
    x = x.clone()
    x[x < 0.5] = 0
    x[x >= 0.5] = 1
    return x


def mask_latents_ref(mask: torch.Tensor, batch_size: int, height: int, width: int) -> torch.Tensor:
    m = F.interpolate(mask, size=(height // 8, width // 8)).to(torch.float16)
    if m.shape[0] < batch_size:
        if batch_size % m.shape[0]:
            raise ValueError("mask batch does not divide the batch")
        m = m.repeat(batch_size // m.shape[0], 1, 1, 1)
    return m


def prepare_inpaint_latents(encode: Callable, image: torch.Tensor, batch_size: int, generator, t_start: int,
                            num_inference_steps: int, strength: float, scaling_factor: float, latent_channels: int = 4,
                            force_upcast: bool = True, dtype=torch.float16):
    """-> (start latents, image latents, noise), each [batch_size, 4, h, w] `dtype`."""
    _, sigmas, ins = euler_tables(num_inference_steps)
    image = image.to(dtype)
    pdt = torch.float32 if force_upcast else dtype
    image = image.to(pdt)
    n_img = image.shape[0]
    if isinstance(generator, list):
        lat = []
        for i in range(n_img):
            mom = encode(image[i:i + 1]).to(pdt)
            eps = _randn((1, latent_channels) + tuple(mom.shape[2:]), generator[i], pdt).to(mom.device)
            lat.append(posterior_sample_ref(mom, eps))
        init = torch.cat(lat, dim=0)
    else:
        mom = encode(image).to(pdt)
        eps = _randn((n_img, latent_channels) + tuple(mom.shape[2:]), generator, pdt).to(mom.device)
        init = posterior_sample_ref(mom, eps)
    image_latents = scaling_factor * init.to(dtype)
    image_latents = image_latents.repeat(batch_size // image_latents.shape[0], 1, 1, 1)
    noise = _randn(image_latents.shape, generator, dtype).to(image_latents.device)
    if strength == 1.0:
        latents = noise * float(ins)
    else:
        latents = add_noise_ref(image_latents, noise, float(sigmas[t_start]))
    return latents, image_latents, noise


@torch.no_grad()
def inpaint_denoise_loop(unet_fn: Callable, latents, image_latents, noise, mask, prompt_embeds, neg_prompt_embeds, pooled,
                         neg_pooled, time_ids, num_inference_steps: int, strength: float, guidance_scale: float = 7.5,
                         set_scale: Optional[Callable[[float], None]] = None, conditioning_scale: float = 1.0,
                         control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                         guidance_rescale: float = 0.0, denoising_end: Optional[float] = None,
                         callback: Optional[Callable] = None, callback_steps: int = 1,
                         trace: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
    """img2img_denoise_loop plus, after every step i of the (truncated) list, the 4-channel blend: the image latents
    re-noised to sigma[t_start + i + 1] (add_noise after step()), the clean image latents after the last step."""
    timesteps, sigmas, _ = euler_tables(num_inference_steps)
    t_start, ts = img2img_timesteps(num_inference_steps, strength)
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
    mask = mask.to(latents.dtype)
    for i in range(n_loop):
        k = t_start + i
        if set_scale is not None:
            off = (i / n_loop < control_guidance_start) or ((i + 1) / n_loop > control_guidance_end)
            set_scale(0.0 if off else conditioning_scale)
        sigma, sigma_next = float(sigmas[k]), float(sigmas[k + 1])
        x2 = torch.cat([latents] * 2) if cfg else latents
        x2 = (x2 / ((sigma ** 2 + 1) ** 0.5)).to(latents.dtype)
        noise_pred = unet_fn(x2, float(timesteps[k]), ehs, text_embeds, tids)
        if cfg:
            u, c = noise_pred.chunk(2)
            eps = u + guidance_scale * (c - u)
            if guidance_rescale > 0.0:
                eps = rescale_noise_cfg(eps, c, guidance_rescale)
        else:
            eps = noise_pred
        x = latents.float()
        x0 = x - (sigma * eps.float()).to(eps.dtype).float()
        latents = (x + (x - x0) / sigma * (sigma_next - sigma)).to(eps.dtype)
        proper = image_latents
        if i < n_loop - 1:
            proper = add_noise_ref(image_latents, noise, float(sigmas[k + 1]))
        latents = (1 - mask) * proper + mask * latents
        if trace is not None:
            trace.append(latents.clone())
        if callback is not None and i % callback_steps == 0:
            callback(i, float(ts[i]), latents)
    return latents


def inpaint_step_ref(noise_pred, latents, sigmas, i: int, guidance: float, image_latents, noise, mask, blend_end: int,
                     use_cfg: bool = True, guidance_rescale: float = 0.0):
    """The rounding points of ih_euler_inpaint_step on fp16 tensors (any device) -> (latents, model_in).

    The kernel is compiled without fast math but with FMA contraction (nvcc's default), like euler_cfg_kernel: the Euler
    update is fma(deriv, sigma_next - sigma, x) and the next-step divisor sqrt(fma(sigma_next, sigma_next, 1)).  Both
    are restated exactly: the product of two fp32 numbers is exact in fp64.  Divisions are by tensors, not by Python
    scalars, because torch multiplies by the reciprocal of a scalar divisor."""
    s, sn = np.float32(sigmas[i]), np.float32(sigmas[i + 1])
    dt = np.float32(sn - s)
    den = np.sqrt(np.float32(np.float64(sn) * np.float64(sn) + 1.0))
    if use_cfg:
        u, c = noise_pred.chunk(2)
        eps = u + guidance * (c - u)
        if guidance_rescale > 0.0:
            eps = rescale_noise_cfg(eps, c, guidance_rescale)
    else:
        eps = noise_pred
    x = latents.float()
    x0 = x - (float(s) * eps.float()).half().float()
    deriv = (x - x0) / torch.full_like(x, float(s))
    xe = (deriv.double() * float(dt) + x.double()).float().half()
    proper = image_latents
    if i + 1 < blend_end:
        proper = image_latents + noise * torch.tensor(float(sn), device=noise.device).half()
    m = mask.half()
    xb = (1 - m) * proper + m * xe
    mi = (xb.float() / torch.full_like(x, float(den))).half()
    return xb, (torch.cat([mi, mi]) if use_cfg else mi)
