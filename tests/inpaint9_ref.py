"""ORACLE (test infrastructure only) for inpainting with the 9-channel SDXL inpainting UNet: CPU restatements of what
[3P] diffusers==0.30.0 `StableDiffusionXLInpaintPipeline` (requirements.txt:25; not vendored) does when
`unet.config.in_channels == 9`.  **Parity unpinned**, like the other [3P] restatements: diffusers is not installable
here and no golden vector exists; they follow the diffusers 0.30.0 sources as published (SURVEY C.32).

* `encode_vae_image_ref`: `_encode_vae_image` -- posterior sample (generator[i] for image i of a list), fp16, scaled;
* `prepare_inpaint9_inputs`: `prepare_latents(return_image_latents=False)` then `prepare_mask_latents`, with their RNG
  order per generator: the image's eps (strength < 1 only: at strength 1 the image is not encoded), the noise, then
  the masked images' eps;
* `unet9_fn`: the model input of every step, cat([scaled latents (CFG halves)], mask, masked-image latents) on dim 1;
  the loops themselves are img2img_ref.img2img_denoise_loop / euler_a_ref.euler_a_denoise_loop (no blend).
"""
from __future__ import annotations

from typing import Callable

import torch

from img2img_ref import _randn, add_noise_ref, posterior_sample_ref
from inpaint_ref import mask_latents_ref
from oracle.scheduler_ref import euler_tables


def encode_vae_image_ref(encode: Callable, image: torch.Tensor, generator, scaling_factor: float,
                         latent_channels: int = 4, force_upcast: bool = True, dtype=torch.float16) -> torch.Tensor:
    image = image.to(dtype)
    pdt = torch.float32 if force_upcast else dtype
    image = image.to(pdt)
    if isinstance(generator, list):
        lat = []
        for i in range(image.shape[0]):
            mom = encode(image[i:i + 1]).to(pdt)
            eps = _randn((1, latent_channels) + tuple(mom.shape[2:]), generator[i], pdt).to(mom.device)
            lat.append(posterior_sample_ref(mom, eps))
        init = torch.cat(lat, dim=0)
    else:
        mom = encode(image).to(pdt)
        eps = _randn((image.shape[0], latent_channels) + tuple(mom.shape[2:]), generator, pdt).to(mom.device)
        init = posterior_sample_ref(mom, eps)
    return scaling_factor * init.to(dtype)


def prepare_inpaint9_inputs(encode: Callable, image: torch.Tensor, mask: torch.Tensor, batch_size: int, generator,
                            t_start: int, num_inference_steps: int, strength: float, scaling_factor: float,
                            latent_channels: int = 4, force_upcast: bool = True, dtype=torch.float16):
    """image [n_img, 3, H, W] in [-1, 1], mask [n_mask, 1, H, W] binarized -> (start latents, mask latents, masked-image
    latents), each with `batch_size` images, `dtype`; CFG halves not formed."""
    _, sigmas, ins = euler_tables(num_inference_steps)
    H, W = image.shape[2:]
    shape = (batch_size, latent_channels, H // 8, W // 8)
    kw = dict(latent_channels=latent_channels, force_upcast=force_upcast, dtype=dtype)
    if strength == 1.0:
        noise = _randn(shape, generator, dtype)
        latents = noise * float(ins)
    else:
        image_latents = encode_vae_image_ref(encode, image, generator, scaling_factor, **kw)
        image_latents = image_latents.repeat(batch_size // image_latents.shape[0], 1, 1, 1)
        noise = _randn(shape, generator, dtype).to(image_latents.device)
        latents = add_noise_ref(image_latents, noise, float(sigmas[t_start]))
    masked_image = image * (mask < 0.5)
    m = mask_latents_ref(mask, batch_size, H, W)
    ml = encode_vae_image_ref(encode, masked_image, generator, scaling_factor, **kw)
    if batch_size % ml.shape[0]:
        raise ValueError("masked image batch does not divide the batch")
    ml = ml.repeat(batch_size // ml.shape[0], 1, 1, 1)
    return latents, m.to(ml.device), ml


def unet9_fn(unet_fn: Callable, mask: torch.Tensor, masked_image_latents: torch.Tensor, cfg: bool) -> Callable:
    """unet_fn of the 4-channel loops for the 9-channel UNet: the scaled latents, then mask, then masked latents."""
    extra = torch.cat([mask, masked_image_latents], dim=1)
    if cfg:
        extra = torch.cat([extra] * 2)
    return lambda x, t, e, te, ti: unet_fn(torch.cat([x, extra.to(x.device, x.dtype)], dim=1), t, e, te, ti)
