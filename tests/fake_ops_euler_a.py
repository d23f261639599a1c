"""TEST-ONLY stand-ins for ops.euler_ancestral_step / ops.euler_ancestral_scale_input in plain PyTorch on the CPU,
used next to tests/fake_ops.py by the Euler Ancestral CPU wiring tests.  They apply the coefficient table and the noise
rows the way the kernel does, on the buffers' own dtype (fp32 in the wiring tests).  Never imported by the product."""
import torch

import fake_ops


def euler_ancestral_step(noise_pred, latents, model_in, coeffs, step_noise, step, guidance, *, use_cfg=True,
                         guidance_rescale=0.0, inpaint=None):
    fake_ops._count[0] += 2
    i = int(step.item())
    sigma, inv_sigma, dt, sigma_up, inv_den_next, sig_next16 = (float(v) for v in coeffs[i, :6])
    if use_cfg:
        u, cond = noise_pred.chunk(2)
        eps = u + guidance * (cond - u)
        if guidance_rescale:
            dims = list(range(1, eps.dim()))
            resc = eps * (cond.std(dim=dims, keepdim=True) / eps.std(dim=dims, keepdim=True))
            eps = guidance_rescale * resc + (1 - guidance_rescale) * eps
    else:
        eps = noise_pred
    x = latents.float()
    x0 = x - sigma * eps.float()
    out = x + (x - x0) * inv_sigma * dt + step_noise[i].float() * sigma_up
    if inpaint is not None:
        image_latents, noise, mask, blend_end = inpaint
        proper = image_latents.float()
        if i + 1 < int(blend_end.item()):
            proper = proper + noise.float() * sig_next16
        m = mask.float()
        out = (1 - m) * proper + m * out
    latents.copy_(out)
    mi = latents.float() * inv_den_next
    model_in.copy_(torch.cat([mi, mi]) if use_cfg else mi)
    step += 1


def euler_ancestral_scale_input(latents, model_in, coeffs, step, duplicate=True):
    fake_ops._count[0] += 1
    mi = latents.float() * float(coeffs[int(step.item()), 6])
    model_in.copy_(torch.cat([mi, mi]) if duplicate else mi)


NAMES = ("euler_ancestral_step", "euler_ancestral_scale_input")
