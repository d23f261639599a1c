"""TEST-ONLY stand-in for ops.dpm_solver_step in plain PyTorch on the CPU, used next to tests/fake_ops.py by the
DPM-Solver++ CPU wiring tests.  It applies the coefficient table the way the kernel does, on the buffers' own dtype
(fp32 in the wiring tests).  Never imported by the product."""
import torch

import fake_ops


def dpm_solver_step(noise_pred, latents, model_in, prev_x0, coeffs, step, loop_begin, guidance, *, use_cfg=True,
                    guidance_rescale=0.0):
    fake_ops._count[0] += 2
    i = int(step.item())
    sigma_s, inv_alpha_s, ratio, c, c_half, inv_r0, first = (float(v) for v in coeffs[i, :7])
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
    x0 = (x - sigma_s * eps.float()) * inv_alpha_s
    out = ratio * x - c * x0
    if not (i == int(loop_begin.item()) or first != 0.0):
        out = out - c_half * (inv_r0 * (x0 - prev_x0.float()))
    latents.copy_(out)
    prev_x0.copy_(x0)
    model_in.copy_(torch.cat([latents, latents]) if use_cfg else latents)
    step += 1


NAMES = ("dpm_solver_step",)
