"""EulerDiscreteScheduler tables for the SDXL-base scheduler_config ([3P] diffusers==0.30.0; the reference calls
set_timesteps / init_noise_sigma / scale_model_input / step at custom_pipelines.py:250,268,334,357), the tables of
EulerAncestralDiscreteScheduler (Euler's, plus a per-step coefficient table; SURVEY A.6), of
DPMSolverMultistepScheduler (DPM-Solver++ 2M, optionally with Karras sigmas; SURVEY A.5) and of UniPCMultistepScheduler
(UniPC bh2 of order 2, optionally with Karras sigmas; SURVEY A.9).

Only the host-side schedule lives here; the per-step arithmetic (scale_model_input, CFG combine, Euler update) is the
fused device kernel `ih_euler_cfg_step` so that a whole denoise step can be replayed as one CUDA graph.  For DPM-Solver++
and UniPC the per-step scalars are evaluated here, once per schedule, into a coefficient table the step kernel
`ih_dpm_solver_step` indexes by the device step counter.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import MappingProxyType
from typing import Any, Mapping

import numpy as np
import torch

from ._lib import IHError

# [3P] SDXL-base scheduler/scheduler_config.json
SDXL_SCHEDULER_CONFIG = {
    "_class_name": "EulerDiscreteScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear", "beta_start": 0.00085,
    "clip_sample": False, "interpolation_type": "linear", "num_train_timesteps": 1000, "prediction_type": "epsilon",
    "sample_max_value": 1.0, "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1,
    "timestep_spacing": "leading", "trained_betas": None, "use_karras_sigmas": False,
}


@dataclass
class EulerSchedule:
    timesteps: np.ndarray        # float32 [T]   (981, 961, ... for T = 50)
    sigmas: np.ndarray           # float32 [T+1] (trailing 0)
    init_noise_sigma: float


class EulerDiscreteScheduler:
    """scaled_linear betas 0.00085 -> 0.012 over 1000 train steps, epsilon prediction, 'leading' spacing, offset 1."""

    order = 1
    kind = "euler"

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        self.num_train_timesteps = num_train_timesteps
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        acp = torch.cumprod(1.0 - betas, dim=0)
        self._sigma_table = (((1 - acp) / acp) ** 0.5).numpy()
        self.steps_offset = steps_offset
        self.schedule: EulerSchedule | None = None
        self._config = MappingProxyType({**SDXL_SCHEDULER_CONFIG, "num_train_timesteps": num_train_timesteps,
                                         "beta_start": beta_start, "beta_end": beta_end, "steps_offset": steps_offset})

    @property
    def config(self) -> Mapping[str, Any]:
        """Read-only diffusers-style config, so that `DPMSolverMultistepScheduler.from_config(pipe.scheduler.config,
        ...)` works as it does with diffusers."""
        return self._config

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


class _FromConfig:
    """diffusers' `<Scheduler>.from_config(config, **overrides)` for a scheduler that implements one configuration:
    the keys of another scheduler's config that this one does not know are ignored, as in diffusers; an override keyword
    it does not know, or a FIXED field at another value, raises IHError.  PARAMS go to the constructor; NO_EFFECT
    fields are accepted and unused.  ALIASES maps a field's values that the diffusers constructor replaces by another
    (e.g. a DPM-Solver++ config's solver_type "midpoint" in UniPC, which registers "bh2") before FIXED is checked, so
    that configs move between schedulers as in diffusers."""

    FIXED: Mapping[str, Any] = {}
    NO_EFFECT: tuple = ()
    PARAMS: tuple = ()
    ALIASES: Mapping[str, Mapping[Any, Any]] = {}

    @classmethod
    def from_config(cls, config: Mapping[str, Any], **overrides):
        name = cls.__name__
        unknown = [k for k in overrides if k not in cls.PARAMS and k not in cls.FIXED and k not in cls.NO_EFFECT]
        if unknown:
            raise IHError(f"{name} does not know {unknown}")
        merged = {**dict(config), **overrides}
        for k, alias in cls.ALIASES.items():
            if k in merged and isinstance(merged[k], str) and merged[k] in alias:
                merged[k] = alias[merged[k]]
        bad = {k: merged[k] for k, v in cls.FIXED.items() if k in merged and merged[k] != v}
        if bad:
            raise IHError(f"{name} implements {({k: cls.FIXED[k] for k in bad})} only, got {bad}")
        return cls(**{k: merged[k] for k in cls.PARAMS if k in merged})


@dataclass
class EulerAncestralSchedule(EulerSchedule):
    coeffs: np.ndarray = None    # float32 [T, EULER_A_COEFFS], the per-step scalars of ih_euler_ancestral_step


EULER_A_COEFFS = 8   # IH_EULER_A_COEFFS: sigma, 1/sigma, dt, sigma_up, 1/den(next), fp16(next sigma), 1/den(sigma), (pad)


class EulerAncestralDiscreteScheduler(_FromConfig, EulerDiscreteScheduler):
    """Euler Ancestral ([3P] diffusers==0.30.0 EulerAncestralDiscreteScheduler with the SDXL-base config: epsilon
    prediction, 'leading' spacing, steps_offset 1).  Restated from the published sources (SURVEY A.6, C.28-C.31);
    parity is unpinned.

    Timesteps, sigmas, init_noise_sigma, scale_model_input and add_noise are Euler's (inherited); only the step differs:
    it moves to sigma_down and adds fresh Gaussian noise times sigma_up, drawn from the pipeline's generator at every
    step.  `set_timesteps` evaluates the per-step scalars with torch fp32 0-dim arithmetic, written as diffusers writes
    it, into `coeffs` (see ih_euler_ancestral_step in include/ih_api.h for the columns)."""

    order = 1
    kind = "euler_a"

    # fields whose other values change the result and have no native implementation (a config asking for Karras sigmas,
    # e.g. a DPM-Solver++ Karras config, is refused rather than silently run with Euler's spacing)
    FIXED = {"beta_schedule": "scaled_linear", "prediction_type": "epsilon", "timestep_spacing": "leading",
             "trained_betas": None, "rescale_betas_zero_snr": False, "use_karras_sigmas": False}
    PARAMS = ("num_train_timesteps", "beta_start", "beta_end", "steps_offset")

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        super().__init__(num_train_timesteps, beta_start, beta_end, steps_offset)
        self._config = MappingProxyType({
            "_class_name": "EulerAncestralDiscreteScheduler", "num_train_timesteps": num_train_timesteps,
            "beta_start": beta_start, "beta_end": beta_end, "steps_offset": steps_offset, **self.FIXED})

    def set_timesteps(self, num_inference_steps: int, device=None) -> EulerAncestralSchedule:
        s = super().set_timesteps(num_inference_steps, device)
        self.schedule = EulerAncestralSchedule(s.timesteps, s.sigmas, s.init_noise_sigma, self._coefficients(s.sigmas))
        return self.schedule

    @staticmethod
    def _coefficients(sigmas: np.ndarray) -> np.ndarray:
        """Row i: the scalars step() and scale_model_input use at schedule index i, each a torch fp32 0-dim tensor
        evaluated as diffusers writes it (the sigmas live on the CPU).  The reciprocals are what ATen multiplies by when
        it divides a CUDA tensor by a 0-dim CPU tensor."""
        sig = torch.from_numpy(sigmas)
        T = len(sigmas) - 1
        out = np.zeros((T, EULER_A_COEFFS), dtype=np.float32)
        for i in range(T):
            sigma_from, sigma_to = sig[i], sig[i + 1]
            sigma_up = (sigma_to**2 * (sigma_from**2 - sigma_to**2) / sigma_from**2) ** 0.5
            sigma_down = (sigma_to**2 - sigma_up**2) ** 0.5
            dt = sigma_down - sigma_from
            row = (sigma_from, 1.0 / sigma_from, dt, sigma_up, 1.0 / ((sigma_to**2 + 1) ** 0.5),
                   sigma_to.half().float(), 1.0 / ((sigma_from**2 + 1) ** 0.5))
            out[i, :7] = [float(v) for v in row]
        return out

    @property
    def coeffs(self):
        return self.schedule.coeffs


@dataclass
class DPMSchedule:
    timesteps: np.ndarray        # int64 [T]
    sigmas: np.ndarray           # float32 [T+1] (trailing 0)
    coeffs: np.ndarray           # float32 [T, DPM_COEFFS or UNIPC_COEFFS], the per-step scalars of ih_dpm_solver_step
    init_noise_sigma: float


DPM_COEFFS = 8       # IH_DPM_COEFFS: sigma_s, 1/alpha_s, sigma_t/sigma_s, c, 0.5*c, 1/r0, first-order flag, (pad)


def _sigma_to_alpha_sigma_t(sigma: torch.Tensor):
    """[3P] DPMSolverMultistepScheduler._sigma_to_alpha_sigma_t: VP alpha and sigma of a Karras-form sigma."""
    alpha_t = 1 / ((sigma**2 + 1) ** 0.5)
    sigma_t = sigma * alpha_t
    return alpha_t, sigma_t


class _VPMultistep(_FromConfig):
    """What DPMSolverMultistepScheduler and UniPCMultistepScheduler share ([3P] diffusers 0.30.0 writes the same
    set_timesteps in both): 'leading' (T + 1) or Karras timesteps, sigmas with a final 0, latents in VP form
    (init_noise_sigma 1, identity scale_model_input) and a per-step coefficient table from `_coefficients`."""

    order = 1                   # [3P] <Scheduler>.order: the callback condition equals Euler's
    init_noise_sigma = 1.0
    PARAMS = ("num_train_timesteps", "beta_start", "beta_end", "steps_offset", "use_karras_sigmas")
    KIND = ""
    EXTRA_CONFIG: Mapping[str, Any] = {}

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1, use_karras_sigmas: bool = False):
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.use_karras_sigmas = bool(use_karras_sigmas)
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.schedule: DPMSchedule | None = None
        self._config = MappingProxyType({
            "_class_name": type(self).__name__, "num_train_timesteps": num_train_timesteps,
            "beta_start": beta_start, "beta_end": beta_end, "steps_offset": steps_offset,
            "use_karras_sigmas": self.use_karras_sigmas, **self.EXTRA_CONFIG, **self.FIXED})

    @property
    def config(self) -> Mapping[str, Any]:
        return self._config

    @property
    def kind(self) -> str:
        return self.KIND + ("_karras" if self.use_karras_sigmas else "")

    def _karras_sigmas_and_timesteps(self, T: int, sig_all: np.ndarray):
        """[3P] _convert_to_karras over the full (flipped) table, rho 7, then _sigma_to_t by log-sigma interpolation."""
        log_sigmas = np.log(sig_all)
        s = np.flip(sig_all).copy()
        sigma_min, sigma_max = s[-1].item(), s[0].item()
        rho = 7.0
        ramp = np.linspace(0, 1, T)
        min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
        sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
        ts = []
        for sigma in sigmas:
            log_sigma = np.log(np.maximum(sigma, 1e-10))
            dists = log_sigma - log_sigmas[:, np.newaxis]
            low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
            high_idx = low_idx + 1
            low, high = log_sigmas[low_idx], log_sigmas[high_idx]
            w = np.clip((low - log_sigma) / (low - high), 0, 1)
            ts.append(((1 - w) * low_idx + w * high_idx).reshape(np.shape(sigma)))
        return sigmas, np.array(ts).round()

    def set_timesteps(self, num_inference_steps: int, device=None) -> DPMSchedule:
        T = int(num_inference_steps)
        n = self.num_train_timesteps
        sig_all = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        if self.use_karras_sigmas:
            sigmas, ts = self._karras_sigmas_and_timesteps(T, sig_all)
        else:
            step_ratio = n // (T + 1)                                   # [3P] 'leading': T + 1, not Euler's T
            ts = (np.arange(0, T + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64) + self.steps_offset
            sigmas = np.interp(ts, np.arange(0, len(sig_all)), sig_all)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)    # final_sigmas_type "zero"
        self.schedule = DPMSchedule(ts.astype(np.int64), sigmas, self._coefficients(sigmas), 1.0)
        return self.schedule

    @property
    def timesteps(self):
        return self.schedule.timesteps

    @property
    def sigmas(self):
        return self.schedule.sigmas

    @property
    def coeffs(self):
        return self.schedule.coeffs


class DPMSolverMultistepScheduler(_VPMultistep):
    """DPM-Solver++ 2M ([3P] diffusers==0.30.0 DPMSolverMultistepScheduler with the SDXL-base config: dpmsolver++,
    solver_order 2, midpoint, epsilon prediction, 'leading' spacing, steps_offset 1, final sigma 0), with or without
    Karras sigmas.  Restated from the published sources (SURVEY A.5, C.22-C.27); parity is unpinned.

    The latents are in VP form, so init_noise_sigma is 1 and scale_model_input is the identity.  Each step is first
    order at the start of the loop and at the last index of the schedule (final sigma 0 forces lower_order_final), second
    order otherwise; `set_timesteps` evaluates every per-step scalar with torch fp32 0-dim arithmetic, written as diffusers
    writes it, into `coeffs` (see ih_dpm_solver_step in include/ih_api.h for the columns)."""

    # fields whose other values change the result and have no native implementation
    FIXED = {"beta_schedule": "scaled_linear", "prediction_type": "epsilon", "algorithm_type": "dpmsolver++",
             "solver_order": 2, "solver_type": "midpoint", "timestep_spacing": "leading", "final_sigmas_type": "zero",
             "thresholding": False, "trained_betas": None, "variance_type": None, "lambda_min_clipped": -math.inf,
             "use_lu_lambdas": False, "use_exponential_sigmas": False, "use_beta_sigmas": False,
             "rescale_betas_zero_snr": False}
    # fields that do not change the result under FIXED (final sigma 0 makes the last step first order either way;
    # the thresholding parameters are unused without thresholding)
    NO_EFFECT = ("lower_order_final", "euler_at_final", "dynamic_thresholding_ratio", "sample_max_value")
    # [3P] DPMSolverMultistepScheduler.__init__ registers solver_type "midpoint" for UniPC's "logrho" / "bh1" / "bh2"
    ALIASES = {"solver_type": {"logrho": "midpoint", "bh1": "midpoint", "bh2": "midpoint"}}
    KIND = "dpmpp_2m"
    EXTRA_CONFIG = {"lower_order_final": True, "euler_at_final": False}

    @staticmethod
    def _coefficients(sigmas: np.ndarray) -> np.ndarray:
        """Row i: the scalars convert_model_output and step use at schedule index i, each a torch fp32 0-dim tensor
        evaluated as diffusers writes it.  1/alpha_s is what ATen multiplies by when it divides an fp16 CUDA tensor by
        the 0-dim CPU alpha_s; 1/r0 is 0 on first-order rows, which never read it."""
        sig = torch.from_numpy(sigmas)
        T = len(sigmas) - 1
        out = np.zeros((T, DPM_COEFFS), dtype=np.float32)
        for i in range(T):
            alpha_t, sigma_t = _sigma_to_alpha_sigma_t(sig[i + 1])
            alpha_s0, sigma_s0 = _sigma_to_alpha_sigma_t(sig[i])
            lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
            lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
            h = lambda_t - lambda_s0
            c = alpha_t * (torch.exp(-h) - 1.0)
            first = i == 0 or i == T - 1
            inv_r0 = torch.zeros((), dtype=torch.float32)
            if not first:
                alpha_s1, sigma_s1 = _sigma_to_alpha_sigma_t(sig[i - 1])
                lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
                h_0 = lambda_s0 - lambda_s1
                r0 = h_0 / h
                inv_r0 = 1.0 / r0
            row = (sigma_s0, 1.0 / alpha_s0, sigma_t / sigma_s0, c, 0.5 * c, inv_r0)
            out[i, :6] = [float(v) for v in row]
            out[i, 6] = 1.0 if first else 0.0
        return out


UNIPC_COEFFS = 16     # IH_UNIPC_COEFFS: see ih_dpm_solver_step (IH_SOLVER_UNIPC_BH2) in include/ih_api.h


def unipc_orders(T: int, begin: int = 0):
    """[3P] UniPCMultistepScheduler.step's order schedule for a loop over indices [begin, T): the predictor's order
    p(i) = min(2, T - i, i - begin + 1) (solver_order 2, lower_order_final, warm-up by lower_order_nums) and the
    corrector's c(i) = p(i - 1), 0 at the loop's first index (no last_sample yet)."""
    p = [min(2, T - i, i - begin + 1) for i in range(T)]
    c = [0 if i <= begin else p[i - 1] for i in range(T)]
    return p, c


class UniPCMultistepScheduler(_VPMultistep):
    """UniPC ([3P] diffusers==0.30.0 UniPCMultistepScheduler with the SDXL-base config: bh2, solver_order 2,
    predict_x0, epsilon prediction, lower_order_final, no disabled corrector, no solver_p, 'leading' spacing,
    steps_offset 1, final sigma 0), with or without Karras sigmas.  Restated from the published sources (SURVEY A.9);
    parity is unpinned.

    Timesteps and sigmas are DPM-Solver++'s.  Each step i first corrects the sample with the new data prediction
    (UniC, order c(i), from step 1 of the loop on), then predicts the next sample (UniP, order p(i)); see
    `unipc_orders`.  `set_timesteps` evaluates every per-step scalar of both, including the fp16 `rhos_c` of the
    order-2 corrector from `torch.linalg.solve`, with torch fp32 0-dim arithmetic written as diffusers writes it, into
    `coeffs` (see ih_dpm_solver_step in include/ih_api.h for the columns)."""

    # fields whose other values change the result and have no native implementation (lower_order_final False would
    # divide by rk = 0 at the final sigma 0)
    FIXED = {"beta_schedule": "scaled_linear", "prediction_type": "epsilon", "solver_order": 2, "solver_type": "bh2",
             "predict_x0": True, "lower_order_final": True, "disable_corrector": [], "solver_p": None,
             "timestep_spacing": "leading", "final_sigmas_type": "zero", "thresholding": False, "trained_betas": None,
             "use_exponential_sigmas": False, "use_beta_sigmas": False, "rescale_betas_zero_snr": False}
    # the thresholding parameters are unused without thresholding
    NO_EFFECT = ("dynamic_thresholding_ratio", "sample_max_value")
    # [3P] UniPCMultistepScheduler.__init__ registers solver_type "bh2" for DPM-Solver's "midpoint" / "heun" / "logrho"
    ALIASES = {"solver_type": {"midpoint": "bh2", "heun": "bh2", "logrho": "bh2"}}
    KIND = "unipc"

    @staticmethod
    def _coefficients(sigmas: np.ndarray) -> np.ndarray:
        """Row i: the scalars convert_model_output, multistep_uni_c_bh_update (sigma_{i-1} -> sigma_i) and
        multistep_uni_p_bh_update (sigma_i -> sigma_{i+1}) use at schedule index i, each a torch fp32 0-dim tensor
        evaluated as diffusers writes it.  Reciprocals are what ATen multiplies by when it divides an fp16 CUDA tensor
        by a 0-dim CPU scalar.  bh2 makes B_h = h_phi_1 = expm1(-h), so alpha_t * B_h is the c column.  Scalars of an
        order a row does not use are 0."""
        sig = torch.from_numpy(sigmas)
        T = len(sigmas) - 1
        p, c = unipc_orders(T)
        out = np.zeros((T, UNIPC_COEFFS), dtype=np.float32)

        def lam(sigma):
            alpha, sigma_vp = _sigma_to_alpha_sigma_t(sigma)
            return torch.log(alpha) - torch.log(sigma_vp)

        def update(s0: int, t: int, order: int, si: int):
            """(sigma_t / sigma_s0, alpha_t * h_phi_1, B_h, hh, rk): rk uses lambda(sigma_si) and is None below order
            2.  bh2 makes B_h = h_phi_1, so alpha_t * h_phi_1 also stands for alpha_t * B_h."""
            alpha_t, sigma_t = _sigma_to_alpha_sigma_t(sig[t])
            alpha_s0, sigma_s0 = _sigma_to_alpha_sigma_t(sig[s0])
            lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
            lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
            h = lambda_t - lambda_s0
            hh = -h
            h_phi_1 = torch.expm1(hh)
            B_h = torch.expm1(hh)
            rk = (lam(sig[si]) - lambda_s0) / h if order == 2 else None
            return sigma_t / sigma_s0, alpha_t * h_phi_1, B_h, hh, rk

        for i in range(T):
            alpha_s, sigma_s = _sigma_to_alpha_sigma_t(sig[i])
            ratio, cc, _, _, rk = update(i, i + 1, p[i], i - 1)
            out[i, :6] = [float(sigma_s), float(1.0 / alpha_s), float(ratio), float(cc),
                          float(1.0 / rk) if p[i] == 2 else 0.0, float(p[i])]
            if c[i] == 0:
                continue
            ratio, cc, B_h, hh, rk = update(i - 1, i, c[i], i - 2)
            if c[i] == 1:
                rho0, rho1 = 0.0, float(torch.tensor([0.5], dtype=torch.float16)[-1])
            else:
                rks = torch.tensor([rk, 1.0])
                h_phi_k = torch.expm1(hh) / hh - 1
                factorial_i = 1
                R, b = [], []
                for k in range(1, c[i] + 1):
                    R.append(torch.pow(rks, k - 1))
                    b.append(h_phi_k * factorial_i / B_h)
                    factorial_i *= k + 1
                    h_phi_k = h_phi_k / hh - 1 / factorial_i
                rhos_c = torch.linalg.solve(torch.stack(R), torch.tensor(b)).to(torch.float16)
                rho0, rho1 = float(rhos_c[0]), float(rhos_c[1])
            out[i, 6:12] = [float(ratio), float(cc), float(1.0 / rk) if c[i] == 2 else 0.0, rho0, rho1, float(c[i])]
        return out


def randn_tensor(shape, generator, dtype: torch.dtype, device, rand_device=None) -> torch.Tensor:
    """N(0, 1) of `shape` and `dtype` on `device`, drawn as [3P] diffusers' randn_tensor draws it, so that a seed gives
    diffusers' numbers: with a list of generators one [1, ...] draw per row, row i with generator[i] on that generator's
    device; otherwise one draw on the generator's device, or on `rand_device` (default `device`) when it is None."""
    if isinstance(generator, list):
        return torch.cat([torch.randn((1,) + tuple(shape[1:]), generator=generator[i], device=generator[i].device,
                                      dtype=dtype).to(device) for i in range(shape[0])])
    dev = generator.device if generator is not None else (rand_device or device)
    return torch.randn(tuple(shape), generator=generator, device=dev, dtype=dtype).to(device)
