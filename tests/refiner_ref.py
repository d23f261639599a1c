"""ORACLE (test infrastructure only) for the SDXL refiner and the base -> refiner handoff.

* `unet_ref(cfg)`: oracle.unet_ref.UNetRef with the mid block built at `cfg.mid_depth` (UNetRef takes the last level's
  depth, which is the base's rule; the refiner's last level has none and its mid block has 4 layers) and diffusers'
  default processors (plain attention over every encoder token) when the config has no image-prompt tokens.
* `begin_step_ref`: a restatement of [3P] diffusers 0.30 StableDiffusionXLImg2ImgPipeline.get_timesteps with
  `denoising_start` (first-order schedulers), on the oracle's Euler timesteps.
* `ensemble_loop`: one denoise loop over the whole schedule that runs one model for the steps before `k` and another
  from `k` on, each with its own conditioning (negative time ids included), Euler or Euler Ancestral; the restated
  ensemble of experts.  Parity **unpinned** like the other [3P] restatements: diffusers is not installable here.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from euler_a_ref import EulerAncestralRef
from oracle.adapter_ref import SelfAttnProcessorRef
from oracle.scheduler_ref import euler_tables
from oracle.unet_ref import MidBlock, UNetRef


def unet_ref(cfg) -> UNetRef:
    ref = UNetRef(cfg)
    if cfg.mid_depth != cfg.transformer_layers_per_block[-1]:
        ref.mid_block = MidBlock(cfg, cfg.block_out_channels[-1], cfg.mid_depth)
    if cfg.num_ip_tokens == 0:
        ref.set_attn_processor({name: SelfAttnProcessorRef() for name in ref.attn_processors})
    return ref


def begin_step_ref(num_inference_steps: int, denoising_start, num_train_timesteps: int = 1000) -> Optional[int]:
    """The schedule index the refiner's loop begins at, or None when `denoising_start` is not a float in (0, 1)
    (diffusers then ignores it).  get_timesteps: t_start = 0, timesteps = scheduler.timesteps;
    cutoff = int(round(N - denoising_start * N)); n = (timesteps < cutoff).sum(); timesteps[-n:]."""
    if not (isinstance(denoising_start, float) and 0 < denoising_start < 1):
        return None
    ts, _, _ = euler_tables(num_inference_steps, num_train_timesteps)
    cutoff = int(round(num_train_timesteps - denoising_start * num_train_timesteps))
    n = int((torch.from_numpy(ts) < cutoff).sum())
    return num_inference_steps - n


@torch.no_grad()
def ensemble_loop(fn_a: Callable, cond_a, fn_b: Callable, cond_b, k: int, latents: torch.Tensor, T: int,
                  guidance_scale: float, ancestral: bool = False, generator=None, begin: int = 0) -> torch.Tensor:
    """Steps [0, k) with `fn_a(sample, t, ehs, text_embeds, time_ids)` and the CFG conditioning `cond_a` = (ehs,
    text_embeds, time_ids) in [negative, positive] order; steps [k, T) with fn_b / cond_b.  Euler steps as in
    oracle.scheduler_ref.denoise_loop, or Euler Ancestral with its noise drawn from `generator` in step order (fp16).
    `begin` > 0 starts at that schedule index from `latents` (the refiner's part alone)."""
    timesteps, sigmas, _ = euler_tables(T)
    sched = EulerAncestralRef(T) if ancestral else None
    for i in range(begin, T):
        fn, (ehs, te, tid) = (fn_a, cond_a) if i < k else (fn_b, cond_b)
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])
        x2 = (torch.cat([latents] * 2) / ((sigma ** 2 + 1) ** 0.5)).to(latents.dtype)
        u, c = fn(x2, float(timesteps[i]), ehs, te, tid).chunk(2)
        eps = u + guidance_scale * (c - u)
        if ancestral:
            sched.step_index = i
            latents = sched.step(eps, latents, generator, noise_dtype=torch.float16)
        else:
            x = latents.float()
            x0 = x - (sigma * eps.float()).to(eps.dtype).float()
            latents = (x + (x - x0) / sigma * (sigma_next - sigma)).to(eps.dtype)
    return latents
