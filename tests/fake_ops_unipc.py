"""TEST-ONLY stand-in for ops.dpm_solver_step in plain PyTorch on the CPU, used next to tests/fake_ops.py by the UniPC
CPU wiring tests.  With `unipc` it applies the coefficient table and the order rule of ih_dpm_solver_step
(IH_SOLVER_UNIPC_BH2) the way the kernel does, on the buffers' own dtype (fp32 in the wiring tests); without it, it is
tests/fake_ops_dpm.py's DPM-Solver++ stand-in.  Never imported by the product."""
import torch

import fake_ops
import fake_ops_dpm


def dpm_solver_step(noise_pred, latents, model_in, prev_x0, coeffs, step, loop_begin, guidance, *, use_cfg=True,
                    guidance_rescale=0.0, unipc=None):
    if unipc is None:
        return fake_ops_dpm.dpm_solver_step(noise_pred, latents, model_in, prev_x0, coeffs, step, loop_begin, guidance,
                                            use_cfg=use_cfg, guidance_rescale=guidance_rescale)
    last_sample, prev_x0_2 = unipc
    fake_ops._count[0] += 2
    i, b = int(step.item()), int(loop_begin.item())
    (sigma_s, inv_alpha_s, p_ratio, p_c, p_inv_rk, p, c_ratio, c_c, c_inv_rk, rho0, rho1,
     c) = (float(v) for v in coeffs[i, :12])
    p, c = min(int(p), i - b + 1), (min(int(c), i - b) if i > b else 0)
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
    m1 = prev_x0.float()
    if c > 0:
        res = (0.5 if c == 1 else rho1) * (x0 - m1)
        if c == 2:
            res = rho0 * (c_inv_rk * (prev_x0_2.float() - m1)) + res
        x = c_ratio * last_sample.float() - c_c * m1 - c_c * res
    out = p_ratio * x - p_c * x0
    if p == 2:
        out = out - p_c * (0.5 * (p_inv_rk * (m1 - x0)))
    prev_x0_2.copy_(prev_x0)
    prev_x0.copy_(x0)
    last_sample.copy_(x)
    latents.copy_(out)
    model_in.copy_(torch.cat([latents, latents]) if use_cfg else latents)
    step += 1


NAMES = ("dpm_solver_step",)
