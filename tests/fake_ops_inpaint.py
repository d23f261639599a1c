"""TEST-ONLY stand-in for ops.euler_inpaint_step in plain PyTorch on the CPU, used next to tests/fake_ops.py and
tests/fake_ops_img2img.py by the inpainting CPU wiring tests.  Never imported by the product."""
import torch

import fake_ops


def euler_inpaint_step(noise_pred, latents, model_in, sigmas, step, guidance, image_latents, noise, mask, blend_end, *,
                       use_cfg=True, guidance_rescale=0.0):
    i = int(step.item())
    fake_ops.euler_step(noise_pred, latents, model_in, sigmas, step, guidance, use_cfg=use_cfg,
                        guidance_rescale=guidance_rescale)
    proper = image_latents
    if i + 1 < int(blend_end.item()):
        proper = image_latents + noise * sigmas[i + 1].to(noise.dtype)
    m = mask.to(latents.dtype)
    latents.copy_((1 - m) * proper + m * latents)
    sn = float(sigmas[i + 1])
    mi = (latents.float() / (sn * sn + 1) ** 0.5).to(model_in.dtype)
    model_in.copy_(torch.cat([mi, mi]) if use_cfg else mi)


NAMES = ("euler_inpaint_step",)
