"""ORACLE (test infrastructure only) for DPM-Solver++ 2M: a CPU / any-device restatement of what [3P]
diffusers==0.30.0 `DPMSolverMultistepScheduler` (requirements.txt:25; not vendored) does with the SDXL-base
scheduler_config, `use_karras_sigmas` either way.  **Parity unpinned**, like the other [3P] restatements: diffusers is
not installable here and the reference holds no golden vector for it; it follows the diffusers 0.30.0 sources as
published (SURVEY A.5, C.22-C.27).  Written independently of imagharmony_b200/scheduler.py:

* `dpm_tables`: set_timesteps ('leading' with T + 1, or Karras over the full sigma table), final sigma 0;
* `step_scalars`: the 0-dim fp32 scalars convert_model_output / step form at one schedule index;
* `DPMSolverRef`: the stateful scheduler (model_outputs, lower_order_nums, step_index) with diffusers' tensor
  expressions, so the dtypes of the tensors it is given decide the rounding points (fp32 oracle, fp16 eager);
* `dpm_denoise_loop`: the loop of custom_pipelines.py:325-363 with this scheduler in place of Euler;
* `dpm_step_ref`: one guided step on given fp16 tensors and history -- the restatement the kernel is tested against.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from oracle.scheduler_ref import rescale_noise_cfg

KNOWN = {   # (T, karras) -> (first three timesteps, last two timesteps, first three sigmas, last three sigmas)
    (20, False): ([941, 894, 847], [95, 48], [10.42505, 8.08818, 6.38031], [0.33262, 0.22041, 0.0]),
    (25, False): ([951, 913, 875], [77, 39], [11.02834, 8.94360, 7.33448], [0.29128, 0.19630, 0.0]),
    (20, True): ([999, 962, 921], [2, 0], [14.61465, 11.72537, 9.34021], [0.04848, 0.02917, 0.0]),
    (25, True): ([999, 970, 938], [1, 0], [14.61465, 12.28304, 10.27783], [0.04374, 0.02917, 0.0]),
}


def _alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def _sigma_to_t(sigma, log_sigmas):
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(np.shape(sigma))


def dpm_tables(num_inference_steps: int, karras: bool = False, num_train_timesteps: int = 1000, steps_offset: int = 1):
    """-> (timesteps int64 [T], sigmas float32 [T+1] with a trailing 0)."""
    acp = _alphas_cumprod(num_train_timesteps)
    sigmas = ((1 - acp) / acp) ** 0.5
    sigmas = sigmas.numpy()
    log_sigmas = np.log(sigmas)
    T = num_inference_steps
    if karras:
        sigmas = np.flip(sigmas).copy()
        sigma_min, sigma_max = sigmas[-1].item(), sigmas[0].item()
        ramp = np.linspace(0, 1, T)
        min_inv_rho, max_inv_rho = sigma_min ** (1 / 7.0), sigma_max ** (1 / 7.0)
        sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** 7.0
        timesteps = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas]).round()
    else:
        step_ratio = num_train_timesteps // (T + 1)
        timesteps = (np.arange(0, T + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
        timesteps += steps_offset
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
    sigmas = np.concatenate([sigmas, [0]]).astype(np.float32)
    return timesteps.astype(np.int64), sigmas


def denoising_end_steps(timesteps, denoising_end: Optional[float], num_train_timesteps: int = 1000) -> int:
    """custom_pipelines.py:307-316 on the DPM timesteps."""
    if denoising_end is None or not isinstance(denoising_end, float) or not 0 < denoising_end < 1:
        return len(timesteps)
    cutoff = int(round(num_train_timesteps - denoising_end * num_train_timesteps))
    return int(sum(1 for t in timesteps if t >= cutoff))


def _alpha_sigma(sigma):
    alpha_t = 1 / ((sigma**2 + 1) ** 0.5)
    sigma_t = sigma * alpha_t
    return alpha_t, sigma_t


def step_scalars(sigmas: torch.Tensor, i: int, second: bool) -> dict:
    """The 0-dim fp32 scalars at schedule index i, evaluated afresh as diffusers' convert_model_output /
    dpm_solver_first_order_update / multistep_dpm_solver_second_order_update write them."""
    alpha_s0, sigma_s0 = _alpha_sigma(sigmas[i])
    alpha_t, sigma_t = _alpha_sigma(sigmas[i + 1])
    lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
    lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
    h = lambda_t - lambda_s0
    out = {"alpha_s": alpha_s0, "sigma_s": sigma_s0, "ratio": sigma_t / sigma_s0,
           "c": alpha_t * (torch.exp(-h) - 1.0)}
    out["c_half"] = 0.5 * (alpha_t * (torch.exp(-h) - 1.0))
    if second:
        alpha_s1, sigma_s1 = _alpha_sigma(sigmas[i - 1])
        lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
        h_0 = lambda_s0 - lambda_s1
        r0 = h_0 / h
        out["inv_r0"] = 1.0 / r0
    return out


class DPMSolverRef:
    """The stateful scheduler.  Scalars are 0-dim fp32 CPU tensors, as in diffusers (self.sigmas lives on the CPU)."""

    def __init__(self, num_inference_steps: int, karras: bool = False):
        ts, sig = dpm_tables(num_inference_steps, karras)
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.from_numpy(sig)
        self.model_outputs: List[Optional[torch.Tensor]] = [None, None]
        self.lower_order_nums = 0
        self.step_index = 0

    def convert_model_output(self, model_output, sample):
        alpha_t, sigma_t = _alpha_sigma(self.sigmas[self.step_index])
        return (sample - sigma_t * model_output) / alpha_t

    def step(self, model_output, sample):
        i = self.step_index
        lower_order_final = i == len(self.timesteps) - 1          # final_sigmas_type "zero"
        model_output = self.convert_model_output(model_output, sample)
        self.model_outputs[0], self.model_outputs[1] = self.model_outputs[1], model_output
        sample = sample.to(torch.float32)                          # "upcast to avoid precision issues"
        if self.lower_order_nums < 1 or lower_order_final:
            k = step_scalars(self.sigmas, i, False)
            prev = k["ratio"] * sample - k["c"] * model_output
        else:
            k = step_scalars(self.sigmas, i, True)
            m0, m1 = self.model_outputs[1], self.model_outputs[0]
            D0, D1 = m0, k["inv_r0"] * (m0 - m1)
            prev = k["ratio"] * sample - k["c"] * D0 - k["c_half"] * D1
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev.to(model_output.dtype)


def _guided(noise_pred, guidance_scale, guidance_rescale, cfg):
    if not cfg:
        return noise_pred
    u, c = noise_pred.chunk(2)
    eps = u + guidance_scale * (c - u)
    if guidance_rescale > 0.0:
        eps = rescale_noise_cfg(eps, c, guidance_rescale)
    return eps


@torch.no_grad()
def dpm_denoise_loop(unet_fn: Callable, latents, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled, time_ids,
                     num_inference_steps: int, karras: bool = False, guidance_scale: float = 5.0,
                     set_scale: Optional[Callable[[float], None]] = None, conditioning_scale: float = 1.0,
                     control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                     guidance_rescale: float = 0.0, denoising_end: Optional[float] = None,
                     callback: Optional[Callable] = None, callback_steps: int = 1) -> torch.Tensor:
    """custom_pipelines.py:296-363 with DPM-Solver++ 2M.  `latents` are the initial noise (init_noise_sigma = 1)."""
    sched = DPMSolverRef(num_inference_steps, karras)
    cfg = guidance_scale > 1.0
    if cfg:
        ehs = torch.cat([neg_prompt_embeds, prompt_embeds], dim=0)
        text_embeds = torch.cat([neg_pooled, pooled], dim=0)
        tids = torch.cat([time_ids, time_ids], dim=0)
    else:
        ehs, text_embeds, tids = prompt_embeds, pooled, time_ids
    T = denoising_end_steps(sched.timesteps.tolist(), denoising_end)
    for i in range(T):
        if set_scale is not None:
            off = (i / T < control_guidance_start) or ((i + 1) / T > control_guidance_end)
            set_scale(0.0 if off else conditioning_scale)
        x2 = torch.cat([latents] * 2) if cfg else latents           # scale_model_input: identity
        t = sched.timesteps[i]
        noise = unet_fn(x2, float(t), ehs, text_embeds, tids)
        latents = sched.step(_guided(noise, guidance_scale, guidance_rescale, cfg), latents)
        if callback is not None and i % callback_steps == 0:
            callback(i, float(t), latents)
    return latents


def dpm_step_ref(noise_pred, latents, prev_x0, num_inference_steps: int, karras: bool, i: int, first: bool,
                 guidance: float, use_cfg: bool = True, guidance_rescale: float = 0.0):
    """Step i of the schedule on the given tensors (any device, fp16 for the kernel test) -> (latents, x0, model_in).
    `first`: the step has no history (the loop starts at i); otherwise `prev_x0` is the previous step's x0."""
    sched = DPMSolverRef(num_inference_steps, karras)
    sched.step_index = i
    sched.lower_order_nums = 0 if first else 1
    sched.model_outputs = [None, prev_x0]
    x = sched.step(_guided(noise_pred, guidance, guidance_rescale, use_cfg), latents)
    return x, sched.model_outputs[1], (torch.cat([x, x]) if use_cfg else x)
