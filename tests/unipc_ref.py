"""ORACLE (test infrastructure only) for UniPC: a CPU / any-device restatement of what [3P] diffusers==0.30.0
`UniPCMultistepScheduler` (not vendored) does with the SDXL-base scheduler_config (bh2, solver_order 2, predict_x0,
epsilon, lower_order_final, 'leading' spacing, final sigma 0), `use_karras_sigmas` either way.  **Parity unpinned**:
diffusers is not installable here and the reference holds no golden vector for it; it follows SURVEY A.9, the recall
of the diffusers 0.30.0 sources.  Written independently of imagharmony_b200/scheduler.py:

* `KNOWN`: known-answer timesteps and sigmas (SURVEY A.9 table);
* `orders`: the predictor / corrector order schedule of `step`;
* `UniPCRef`: the stateful scheduler (model_outputs, timestep_list, last_sample, lower_order_nums, this_order,
  step_index) with diffusers' tensor expressions -- `multistep_uni_c_bh_update`, `multistep_uni_p_bh_update`,
  `torch.linalg.solve`, `einsum` -- so the dtypes of the tensors it is given decide the rounding points (fp32 oracle,
  fp16 eager);
* `unipc_denoise_loop`: the loop of custom_pipelines.py:325-363 with this scheduler in place of Euler;
* `unipc_step_ref`: one guided step on given fp16 tensors and history -- the restatement the kernel is tested against.

The timesteps / sigmas are DPM-Solver++'s (diffusers writes the same set_timesteps in both), so `dpm_tables` of
tests/dpm_ref.py is reused for them.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch

from dpm_ref import _guided, denoising_end_steps, dpm_tables

KNOWN = {   # (T, karras) -> (first three timesteps, last two timesteps, first three sigmas, last three sigmas)
    (10, False): ([901, 811, 721], [181, 91], [8.39069, 5.37634, 3.63065], [0.52698, 0.32353, 0.0]),
    (20, False): ([941, 894, 847], [95, 48], [10.42505, 8.08818, 6.38031], [0.33262, 0.22041, 0.0]),
    (25, False): ([951, 913, 875], [77, 39], [11.02834, 8.94360, 7.33448], [0.29128, 0.19630, 0.0]),
    (10, True): ([999, 916, 815], [7, 0], [14.61465, 9.10294, 5.47840], [0.08191, 0.02917, 0.0]),
    (20, True): ([999, 962, 921], [2, 0], [14.61465, 11.72537, 9.34021], [0.04848, 0.02917, 0.0]),
    (25, True): ([999, 970, 938], [1, 0], [14.61465, 12.28304, 10.27783], [0.04374, 0.02917, 0.0]),
}


def orders(T: int, begin: int = 0):
    """(predictor orders, corrector orders) by schedule index for a loop over [begin, T), as `step` forms them: the
    predictor's this_order = min(solver_order, T - i) capped by lower_order_nums + 1; the corrector runs from the
    second step of the loop on, with the previous step's this_order."""
    p, c = [0] * T, [0] * T
    lower = 0
    for i in range(begin, T):
        c[i] = p[i - 1] if i > begin else 0
        p[i] = min(min(2, T - i), lower + 1)
        lower = min(lower + 1, 2)
    return p, c


def _alpha_sigma(sigma):
    alpha_t = 1 / ((sigma**2 + 1) ** 0.5)
    sigma_t = sigma * alpha_t
    return alpha_t, sigma_t


class UniPCRef:
    """The stateful scheduler.  Scalars are 0-dim fp32 CPU tensors, as in diffusers (self.sigmas lives on the CPU)."""

    def __init__(self, num_inference_steps: int, karras: bool = False):
        ts, sig = dpm_tables(num_inference_steps, karras)
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.from_numpy(sig)
        self.model_outputs: List[Optional[torch.Tensor]] = [None, None]
        self.timestep_list: List = [None, None]
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = None
        self.step_index = 0
        self.disable_corrector: list = []

    def convert_model_output(self, model_output, sample):
        alpha_t, sigma_t = _alpha_sigma(self.sigmas[self.step_index])
        return (sample - sigma_t * model_output) / alpha_t

    def _rks_b(self, h, lambda_s0, order, first_si, model_output_list, m0):
        rks, D1s = [], []
        for i in range(1, order):
            si = first_si - (i - 1)
            mi = model_output_list[-(i + 1)]
            alpha_si, sigma_si = _alpha_sigma(self.sigmas[si])
            lambda_si = torch.log(alpha_si) - torch.log(sigma_si)
            rk = (lambda_si - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(1.0)
        rks = torch.tensor(rks, device=m0.device)
        hh = -h
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = torch.expm1(hh)                                   # bh2
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        R = torch.stack(R)
        b = torch.tensor(b, device=m0.device)
        return D1s, R, b, h_phi_1, B_h

    def multistep_uni_p_bh_update(self, sample, order):
        model_output_list = self.model_outputs
        m0 = model_output_list[-1]
        x = sample
        sigma_t, sigma_s0 = self.sigmas[self.step_index + 1], self.sigmas[self.step_index]
        alpha_t, sigma_t = _alpha_sigma(sigma_t)
        alpha_s0, sigma_s0 = _alpha_sigma(sigma_s0)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        D1s, R, b, h_phi_1, B_h = self._rks_b(h, lambda_s0, order, self.step_index - 1, model_output_list, m0)
        if len(D1s) > 0:
            D1s = torch.stack(D1s, dim=1)
            rhos_p = torch.tensor([0.5], dtype=x.dtype, device=x.device)     # order 2
        else:
            D1s = None
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        pred_res = torch.einsum("k,bkc...->bc...", rhos_p, D1s) if D1s is not None else 0
        x_t = x_t_ - alpha_t * B_h * pred_res
        return x_t.to(x.dtype)

    def multistep_uni_c_bh_update(self, this_model_output, last_sample, this_sample, order):
        model_output_list = self.model_outputs
        m0 = model_output_list[-1]
        x = last_sample
        model_t = this_model_output
        sigma_t, sigma_s0 = self.sigmas[self.step_index], self.sigmas[self.step_index - 1]
        alpha_t, sigma_t = _alpha_sigma(sigma_t)
        alpha_s0, sigma_s0 = _alpha_sigma(sigma_s0)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        D1s, R, b, h_phi_1, B_h = self._rks_b(h, lambda_s0, order, self.step_index - 2, model_output_list, m0)
        D1s = torch.stack(D1s, dim=1) if len(D1s) > 0 else None
        if order == 1:
            rhos_c = torch.tensor([0.5], dtype=x.dtype, device=x.device)
        else:
            rhos_c = torch.linalg.solve(R, b).to(x.device).to(x.dtype)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        corr_res = torch.einsum("k,bkc...->bc...", rhos_c[:-1], D1s) if D1s is not None else 0
        D1_t = model_t - m0
        x_t = x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * D1_t)
        return x_t.to(x.dtype)

    def step(self, model_output, sample, correct: bool = True):
        """`correct=False` skips the corrector (the test that it matters)."""
        use_corrector = (self.step_index > 0 and self.step_index - 1 not in self.disable_corrector
                         and self.last_sample is not None and correct)
        model_output_convert = self.convert_model_output(model_output, sample)
        if use_corrector:
            sample = self.multistep_uni_c_bh_update(model_output_convert, self.last_sample, sample, self.this_order)
        self.model_outputs[0] = self.model_outputs[1]
        self.timestep_list[0] = self.timestep_list[1]
        self.model_outputs[-1] = model_output_convert
        self.timestep_list[-1] = self.timesteps[self.step_index]
        this_order = min(2, len(self.timesteps) - self.step_index)          # lower_order_final
        self.this_order = min(this_order, self.lower_order_nums + 1)
        self.last_sample = sample
        prev_sample = self.multistep_uni_p_bh_update(sample, self.this_order)
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev_sample


@torch.no_grad()
def unipc_denoise_loop(unet_fn: Callable, latents, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled, time_ids,
                       num_inference_steps: int, karras: bool = False, guidance_scale: float = 5.0,
                       set_scale: Optional[Callable[[float], None]] = None, conditioning_scale: float = 1.0,
                       control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                       guidance_rescale: float = 0.0, denoising_end: Optional[float] = None,
                       callback: Optional[Callable] = None, callback_steps: int = 1,
                       correct: bool = True) -> torch.Tensor:
    """custom_pipelines.py:296-363 with UniPC.  `latents` are the initial noise (init_noise_sigma = 1)."""
    sched = UniPCRef(num_inference_steps, karras)
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
        latents = sched.step(_guided(noise, guidance_scale, guidance_rescale, cfg), latents, correct=correct)
        if callback is not None and i % callback_steps == 0:
            callback(i, float(t), latents)
    return latents


def unipc_step_ref(noise_pred, latents, last_sample, prev_x0, prev_x0_2, num_inference_steps: int, karras: bool,
                   i: int, begin: int, guidance: float, use_cfg: bool = True, guidance_rescale: float = 0.0):
    """Step i of a loop that began at schedule index `begin`, on the given tensors (any device, fp16 for the kernel
    test) -> (latents, last_sample, prev_x0, prev_x0_2, model_in).  The history is what the loop's earlier steps left:
    `last_sample` the corrected sample of step i - 1, `prev_x0` / `prev_x0_2` the data predictions of steps i - 1 and
    i - 2; the scheduler state (orders, lower_order_nums) is that of step i of the loop."""
    T = num_inference_steps
    sched = UniPCRef(T, karras)
    p, _ = orders(T, begin)
    sched.step_index = i
    sched.lower_order_nums = min(i - begin, 2)
    sched.model_outputs = [prev_x0_2, prev_x0]
    sched.last_sample = last_sample if i > begin else None
    sched.this_order = p[i - 1] if i > begin else None
    x = sched.step(_guided(noise_pred, guidance, guidance_rescale, use_cfg), latents)
    return x, sched.last_sample, sched.model_outputs[1], sched.model_outputs[0], (torch.cat([x, x]) if use_cfg else x)


def step_scalars(sigmas: torch.Tensor, i: int, p: int, c: int) -> dict:
    """The 0-dim fp32 scalars at schedule index i for predictor order p and corrector order c (0: no corrector),
    evaluated afresh as diffusers' convert_model_output / multistep_uni_c_bh_update / multistep_uni_p_bh_update write
    them; `rhos_c` is the fp16 tensor of the corrector."""
    ref = UniPCRef.__new__(UniPCRef)
    ref.sigmas = sigmas
    alpha_s, sigma_s = _alpha_sigma(sigmas[i])
    out = {"sigma_s": sigma_s, "inv_alpha_s": 1.0 / alpha_s}
    for name, s0, t, order, first_si in (("p", i, i + 1, p, i - 1), ("c", i - 1, i, c, i - 2)):
        if order == 0:
            continue
        alpha_t, sigma_t = _alpha_sigma(sigmas[t])
        alpha_s0, sigma_s0 = _alpha_sigma(sigmas[s0])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        m = [torch.zeros(1), torch.zeros(1)]
        D1s, R, b, h_phi_1, B_h = ref._rks_b(h, lambda_s0, order, first_si, m, m[-1])
        out[name + "_ratio"] = sigma_t / sigma_s0
        out[name + "_c"] = alpha_t * h_phi_1
        out[name + "_aB"] = alpha_t * B_h
        if order == 2:
            alpha_si, sigma_si = _alpha_sigma(sigmas[first_si])
            out[name + "_inv_rk"] = 1.0 / ((torch.log(alpha_si) - torch.log(sigma_si) - lambda_s0) / h)
        if name == "c":
            out["rhos_c"] = (torch.tensor([0.5], dtype=torch.float16) if order == 1
                             else torch.linalg.solve(R, b).to(torch.float16))
    return out
