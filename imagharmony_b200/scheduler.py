"""EulerDiscreteScheduler tables for the SDXL-base scheduler_config ([3P] diffusers==0.30.0; the reference calls
set_timesteps / init_noise_sigma / scale_model_input / step at custom_pipelines.py:250,268,334,357).

Only the host-side schedule lives here; the per-step arithmetic (scale_model_input, CFG combine, Euler update) is the
fused device kernel `ih_euler_cfg_step` so that a whole denoise step can be replayed as one CUDA graph.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch


@dataclass
class EulerSchedule:
    timesteps: np.ndarray        # float32 [T]   (981, 961, ... for T = 50)
    sigmas: np.ndarray           # float32 [T+1] (trailing 0)
    init_noise_sigma: float


class EulerDiscreteScheduler:
    """scaled_linear betas 0.00085 -> 0.012 over 1000 train steps, epsilon prediction, 'leading' spacing, offset 1."""

    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        self.num_train_timesteps = num_train_timesteps
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        acp = torch.cumprod(1.0 - betas, dim=0)
        self._sigma_table = (((1 - acp) / acp) ** 0.5).numpy()
        self.steps_offset = steps_offset
        self.schedule: EulerSchedule | None = None

    def set_timesteps(self, num_inference_steps: int, device=None) -> EulerSchedule:
        n = self.num_train_timesteps
        ratio = n // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.float32) + self.steps_offset
        sig = np.interp(ts, np.arange(0, n), self._sigma_table)
        sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.schedule = EulerSchedule(ts.astype(np.float32), sigmas, float((sigmas.max() ** 2 + 1) ** 0.5))
        return self.schedule

    @staticmethod
    def img2img_begin_index(num_inference_steps: int, strength: float) -> int:
        """[3P] StableDiffusionXLImg2ImgPipeline.get_timesteps: an image-to-image run of `strength` skips the first
        t_start entries of the schedule and denoises over timesteps[t_start:] (the scheduler's begin index)."""
        init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
        return max(num_inference_steps - init_timestep, 0)

    def add_noise_sigma(self, begin_index: int) -> float:
        """The sigma EulerDiscreteScheduler.add_noise scales the noise with before the first image-to-image step."""
        return float(self.sigmas[begin_index])

    @property
    def timesteps(self):
        return self.schedule.timesteps

    @property
    def sigmas(self):
        return self.schedule.sigmas

    @property
    def init_noise_sigma(self) -> float:
        return self.schedule.init_noise_sigma
