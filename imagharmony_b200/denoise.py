"""The denoise loop of custom_pipelines.py:325-363 as a device-resident loop.

One step = UNet forward on the scaled (CFG) batch + the fused guidance/Euler kernel; everything a step needs (timestep,
sigma pair, step index) is read from device memory, so the step is captured ONCE as a CUDA graph and replayed T times
with no host work in between.  Step-invariant work (cross-attention K/V of all 70 attn2 layers, the text_time
embedding) runs once per call in `prepare`.

Loop options of the reference that are honoured here (all graph-replayed; a callback only breaks the replay sequence,
not the graph): classifier-free guidance on or off (`guidance_scale <= 1`, :223,:332,:348), `guidance_rescale`
(:352-354), `denoising_end` (:307-316, via `num_loop_steps`), `callback` / `callback_steps` (:359-363),
`control_guidance_start/end` IP-scale gating (:326-329), negative micro-conditioning time ids (:286-300).

Schedulers: EulerDiscreteScheduler (the reference's), EulerAncestralDiscreteScheduler (SURVEY A.6) and
DPMSolverMultistepScheduler (DPM-Solver++ 2M, SURVEY A.5), chosen by the engine's scheduler object in one place of `run`.
The DPM step reads its per-step scalars from a coefficient table and the previous step's data prediction from a static
`prev_x0` buffer, both device-resident, so it too is one graph per shape.  The Euler Ancestral step reads its scalars
from a coefficient table and its Gaussian noise from row `step` of a static [T, n, 4, h, w] buffer that `run` fills from
the caller's generator(s) before the replays, outside any capture: the draws are torch's, in diffusers' order, so a seed
gives diffusers' noise (a Philox stream inside the kernel would not reproduce torch's generator).

`run` refuses a call (IHError) before it allocates, copies or launches anything, so a refused call leaves no buffer
and no K/V projection behind.  A validated call is described by one `_Loop` record, which `_step`, `_capture` and
`_first_input` read.

Graph lifetime: a captured graph holds raw pointers.  Everything it reads lives in buffers that are owned per shape
and never freed while the graph exists -- the engine's static buffers (`_pool`, keyed by buffer name and shape) and
schedule tables (`_schedules`), the processors' K/V buffers and the UNet's add-embedding buffer (per-shape dicts inside
those objects), and the library's grow-only scratch buffers whose re-allocation bumps `ops.workspace_generation()`.  A
graph is replayed only if it was captured under the current UNet `graph_epoch` (weights / processors unchanged) and the
current workspace generation; otherwise it is re-captured; a graph with ControlNets also needs each of its nets to be
the object, at the `graph_epoch`, it was captured with (tracked per net index, so reloading one net re-captures only
the graphs that contain it).

ControlNet (`run(controlnet=...)`): a step runs the active ControlNets' forwards in net order, then the UNet with
their residuals summed and injected after the mid block in one launch, then the unchanged step kernel, all in the one
graph.  There is one graph per distinct set of active nets (staggered windows of K nets give at most 2K + 1); steps
where no net is active (keep[i] = 0 for all) replay the ControlNet-free graph.  The scale vectors are read from device
memory, so a new controlnet_conditioning_scale does not re-capture.

T2I-Adapter (`run(adapter=...)`): the adapter runs once per call, outside the loop (the pipeline's job); its four
features are copied into static buffers and its scale into a device value, and the step graph with the features adds
them inside the UNet's encoder (4 launches).  Steps past the adapter's window (keep[i] = 0) replay the plain graph.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple, Union

import numpy as np
import torch

from . import ops
from ._lib import IH_CN_MAX_NETS, IHError
from .controlnet import controlnet_scales
from .scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler, EulerDiscreteScheduler,
                        randn_tensor)
from .t2i_adapter import AdapterCall
from .unet import UNet2DConditionModel, require_adapter_shapes, require_latent_size

# option -> the options it cannot be combined with, and why
_EXCLUDES = (
    ("DPMSolverMultistepScheduler", ("begin_step", "inpaint", "unet_cond", "start_step", "stop_after"),
     "it runs whole text-to-image loops; EulerDiscreteScheduler and EulerAncestralDiscreteScheduler support these "
     "options"),
    ("unet_cond", ("inpaint", "start_step", "stop_after"), "the 9-channel UNet is not blended and resumes nothing"),
    ("controlnet", ("begin_step", "inpaint", "unet_cond", "start_step", "stop_after"), "it runs text-to-image loops"),
    ("inpaint", ("start_step", "stop_after"), "inpainting resumes nothing"),
    ("begin_step", ("start_step", "stop_after"), "image-to-image resumes nothing"),
    ("adapter", ("begin_step", "inpaint", "unet_cond", "controlnet", "start_step", "stop_after"),
     "the T2I-Adapter runs text-to-image loops (diffusers has no SDXL pipeline for these combinations)"),
)


class GraphKey(NamedTuple):
    """The key of one captured step graph (DenoiseEngine._graphs).  Read it by field name.  It is also a plain tuple,
    and fields added later go before `cond`, so the positions of the older fields stay where they were (the shape in
    front, `ib` second to last, `controlnet` last)."""
    n: int
    h: int
    w: int
    L: int
    T: int
    use_cfg: bool
    guidance: float
    rescale: float
    scale: float                              # the IP scale of the step
    kind: str                                 # the scheduler's
    adapter: bool                             # T2I-Adapter features added
    cond: bool                                # 9-channel UNet
    ib: bool                                  # 4-channel inpainting blend
    controlnet: Optional[tuple]               # ("controlnet", guess mode with CFG, active net indices) or None


@dataclass
class _Loop:
    """One validated call's step: its static buffers, tables and options, and whichever scheduler / conditioning
    parts apply (None where they do not)."""
    st: dict                                  # DenoiseEngine._buffers
    timesteps: torch.Tensor
    sigmas: torch.Tensor
    guidance: float
    use_cfg: bool
    rescale: float
    shape: Tuple[int, int, int, int, int]     # (n, h, w, L, T)
    kind: str                                 # the scheduler's
    coeffs: Optional[torch.Tensor] = None     # DPM-Solver++ / Euler Ancestral coefficient table
    dpm: Optional[dict] = None                # DPM-Solver++: prev_x0, loop_begin
    noise: Optional[torch.Tensor] = None      # Euler Ancestral step noise [T, n, C, h, w]
    ib: Optional[dict] = None                 # 4-channel inpainting: image_latents, noise, mask, blend_end
    cond: Optional[torch.Tensor] = None       # 9-channel UNet: mask | masked-image latents
    adapter: Optional[tuple] = None           # T2I-Adapter: (static feature buffers, device fp32 scale)

    def graph_key(self, scale: float, cn, adapter: bool = False) -> "GraphKey":
        """The key of the step graph with IP scale `scale`, active ControlNet step `cn` (see DenoiseEngine._step) and
        the T2I-Adapter's features added or not."""
        return GraphKey(*self.shape, self.use_cfg, self.guidance, self.rescale, scale, self.kind, bool(adapter),
                        self.cond is not None, self.ib is not None,
                        None if cn is None else ("controlnet", cn[2] > 0, cn[0]))


class DenoiseEngine:
    def __init__(self, unet: UNet2DConditionModel, use_cuda_graph: bool = True,
                 scheduler: Optional[Union[EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                                           DPMSolverMultistepScheduler]] = None):
        self.unet = unet
        self.device = unet.conv_in.weight.device
        self.scheduler = scheduler or EulerDiscreteScheduler()      # the pipeline's own scheduler object when given
        self.use_cuda_graph = use_cuda_graph and self.device.type == "cuda"
        self._graphs: Dict[GraphKey, Tuple[torch.cuda.CUDAGraph, int]] = {}   # key -> (graph, workspace generation)
        self._pool: Dict[Tuple[str, Tuple], torch.Tensor] = {}         # (buffer name, shape key) -> static buffer
        # (kind, T) -> (timesteps fp32, sigmas fp32, init_noise_sigma, coefficient table or None)
        self._schedules: Dict[Tuple[str, int], tuple] = {}
        # net index -> (ControlNet, graph_epoch) the graphs with that net were captured for.  The model object itself is
        # kept, not its id: a freed model's id can be reused by a new one that reaches the same epoch
        self._cn_epochs: Dict[int, Tuple] = {}
        self._epoch = getattr(unet, "graph_epoch", 0)
        self._loop: Optional[_Loop] = None                              # the last call's
        self.last_launches_per_step = 0
        self.graphs_captured = 0

    # ------------------------------------------------------------------------------------------------------------
    def _schedule(self, num_steps: int) -> tuple:
        key = (self.scheduler.kind, num_steps)
        t = self._schedules.get(key)
        if t is None:
            s = self.scheduler.set_timesteps(num_steps)
            coeffs = getattr(s, "coeffs", None)
            t = (torch.from_numpy(s.timesteps.astype(np.float32)).to(self.device),
                 torch.from_numpy(s.sigmas).to(self.device), s.init_noise_sigma,
                 None if coeffs is None else torch.from_numpy(coeffs).to(self.device))
            self._schedules[key] = t
        return t

    def tables(self, num_steps: int):
        """(timesteps fp32, sigmas fp32, init_noise_sigma) of the engine's scheduler on the device."""
        return self._schedule(num_steps)[:3]

    def coeffs(self, num_steps: int) -> torch.Tensor:
        """The DPM-Solver++ / Euler Ancestral coefficient table on the device."""
        return self._schedule(num_steps)[3]

    def set_scale(self, scale: float) -> None:
        """IPAdapter.set_scale / pipeline.set_scale (ip_adapter.py:179-182, custom_pipelines.py:17-20)."""
        for p in self.unet.attn_processors.values():
            if hasattr(p, "to_k_ip"):
                p.scale = scale

    def invalidate_graphs(self) -> None:
        self._graphs.clear()

    def _buf(self, name: str, key: tuple, shape, dtype=torch.float16, zero: bool = False) -> torch.Tensor:
        """The static buffer `name` for shape key `key`, allocated on first use and never freed (the graph-lifetime rule
        above).  `zero` fills a new one with zeros, so that a capture's warm-up step reads finite values."""
        buf = self._pool.get((name, key))
        if buf is None:
            buf = torch.empty(shape, dtype=dtype, device=self.device)
            if zero:
                buf.zero_()
            self._pool[(name, key)] = buf
        return buf

    def _buffers(self, n: int, h: int, w: int, L: int, use_cfg: bool = True) -> dict:
        """The step's static inputs and state per (n, h, w, L, use_cfg)."""
        cfg, key, b = self.unet.config, (n, h, w, L, use_cfg), 2 * n if use_cfg else n
        return {"latents": self._buf("latents", key, (n, cfg.out_channels, h, w)),
                "model_in": self._buf("model_in", key, (b, cfg.out_channels, h, w)),
                "ehs": self._buf("ehs", key, (b, L, cfg.cross_attention_dim)),
                "text_embeds": self._buf("text_embeds", key, (b, cfg.pooled_embed_dim)),
                "time_ids": self._buf("time_ids", key, (b, cfg.num_time_ids), torch.float32),
                "step": self._buf("step", key, (1,), torch.int32, zero=True)}

    def _draw_ancestral_noise(self, buf: torch.Tensor, generator, begin: int, end: int) -> None:
        """Rows [begin, end) of the step noise, one draw per step in step order, as [3P] diffusers' randn_tensor draws
        it inside EulerAncestralDiscreteScheduler.step: fp16, shaped like the guided prediction, from the device's
        default generator when `generator` is None."""
        for i in range(begin, end):
            buf[i].copy_(randn_tensor(buf.shape[1:], generator, torch.float16, self.device))

    def _first_input(self, loop: _Loop) -> None:
        """The UNet input of the loop's first step from st["latents"] (custom_pipelines.py:332-334)."""
        st = loop.st
        if loop.noise is not None:   # the convention of the ancestral kernel's later inputs: x * fp32(1 / sqrt(s^2 + 1))
            ops.euler_ancestral_scale_input(st["latents"], st["model_in"], loop.coeffs, st["step"],
                                            duplicate=loop.use_cfg)
        elif loop.dpm is None:
            ops.scale_model_input(st["latents"], st["model_in"], loop.sigmas, st["step"], duplicate=loop.use_cfg)
        else:                                        # DPM-Solver++: scale_model_input is the identity
            n = st["latents"].shape[0]
            st["model_in"][:n].copy_(st["latents"])
            if loop.use_cfg:
                st["model_in"][n:].copy_(st["latents"])

    def _restart(self, loop: _Loop, latents: torch.Tensor, step: int) -> None:
        """Puts the loop at its start: `latents`, the step counter at `step` and the first step's UNet input."""
        loop.st["latents"].copy_(latents, non_blocking=True)
        loop.st["step"].fill_(step)
        self._first_input(loop)

    def _step(self, loop: _Loop, cn=None, adapter: bool = False):
        st, residuals = loop.st, None
        if cn is not None:          # (active net indices, [(ControlNet, emb, scale)], first image they run on)
            _, nets, b0 = cn
            outs = [model(st["model_in"][b0:], loop.timesteps, st["ehs"][b0:], text_embeds=st["text_embeds"][b0:],
                          time_ids=st["time_ids"][b0:], step=st["step"], cond_embedding=emb, scale=scale)
                    for model, emb, scale in nets]
            residuals = (outs[0] if len(outs) == 1 else outs, b0)
        noise = self.unet(st["model_in"], loop.timesteps, st["ehs"], st["text_embeds"], st["time_ids"], step=st["step"],
                          cond=loop.cond, controlnet_residuals=residuals,
                          adapter_residuals=loop.adapter if adapter else None)
        ib = loop.ib
        if loop.dpm is not None:
            ops.dpm_solver_step(noise, st["latents"], st["model_in"], loop.dpm["prev_x0"], loop.coeffs, st["step"],
                                loop.dpm["loop_begin"], loop.guidance, use_cfg=loop.use_cfg,
                                guidance_rescale=loop.rescale)
        elif loop.noise is not None:
            blend = None if ib is None else (ib["image_latents"], ib["noise"], ib["mask"], ib["blend_end"])
            ops.euler_ancestral_step(noise, st["latents"], st["model_in"], loop.coeffs, loop.noise, st["step"],
                                     loop.guidance, use_cfg=loop.use_cfg, guidance_rescale=loop.rescale, inpaint=blend)
        elif ib is None:
            ops.euler_step(noise, st["latents"], st["model_in"], loop.sigmas, st["step"], loop.guidance,
                           use_cfg=loop.use_cfg, guidance_rescale=loop.rescale)
        else:
            ops.euler_inpaint_step(noise, st["latents"], st["model_in"], loop.sigmas, st["step"], loop.guidance,
                                   ib["image_latents"], ib["noise"], ib["mask"], ib["blend_end"], use_cfg=loop.use_cfg,
                                   guidance_rescale=loop.rescale)

    # ------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def run(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, negative_prompt_embeds: Optional[torch.Tensor],
            pooled: torch.Tensor, negative_pooled: Optional[torch.Tensor], time_ids: torch.Tensor,
            num_inference_steps: int, guidance_scale: float = 5.0, ip_scale: float = 1.0,
            control_guidance_start: float = 0.0, control_guidance_end: float = 1.0, stop_after: Optional[int] = None,
            start_step: int = 0, guidance_rescale: float = 0.0, num_loop_steps: Optional[int] = None,
            callback: Optional[Callable] = None, callback_steps: int = 1,
            negative_time_ids: Optional[torch.Tensor] = None, begin_step: int = 0,
            inpaint: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
            generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
            unet_cond: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, controlnet=None,
            adapter: Optional[AdapterCall] = None) -> torch.Tensor:
        """latents [n,4,h,w] (already scaled by init_noise_sigma; host or device); embeds host or device tensors.
        Returns the latents after the last executed step as a new device tensor.

        `stop_after` stops after step index k - 1 (PNS preview); `start_step` = k resumes a trajectory whose `latents`
        are the output of a `stop_after=k` call with the same schedule (two-phase PNS: preview all candidates,
        continue only the winner).  `num_loop_steps` = k truncates the timestep list to its first k entries the way
        `denoising_end` does (custom_pipelines.py:307-316: the gating fractions of :326 then use k, the sigma table
        stays the full schedule's).  `guidance_scale <= 1` runs the UNet on the positive branch only (:223).

        `begin_step` = k is image-to-image ([3P] StableDiffusionXLImg2ImgPipeline): the loop runs over the schedule's
        entries [k, num_loop_steps) starting from `latents` that already carry the noise of sigma[k]; the device step
        counter starts at k, and the gating fractions and callback indices count from k, i.e. they see the truncated
        list.  It resumes nothing, so it cannot be combined with `start_step` / `stop_after` (IHError).  The step graphs
        do not depend on k: image-to-image replays the text-to-image graphs of the same shape.

        `inpaint` = (image_latents [n,4,h,w], noise [n,4,h,w], mask [n,1,h,w]) is inpainting with a 4-channel UNet
        ([3P] StableDiffusionXLInpaintPipeline): after every step the latents outside the mask are replaced by the
        image latents re-noised to the next sigma, and by the clean image latents after the last step of the loop
        (ops.euler_inpaint_step).  It composes with begin_step, num_loop_steps and the other loop options, not with
        start_step / stop_after (IHError).  Its step graphs are captured once per shape next to the text-to-image
        ones; the loop end is a device value, so they serve every num_loop_steps.

        With a DPMSolverMultistepScheduler the loop is DPM-Solver++ 2M: the first model input is the latents themselves,
        and every step updates the latents and the previous data prediction on the device.  It runs whole
        text-to-image loops, with every option above except begin_step, inpaint, start_step and stop_after (IHError):
        they would need the VP-form add_noise, or the history of another call.

        `unet_cond` = (mask [n,1,h,w], masked_image_latents [n,4,h,w]) is inpainting with the 9-channel inpainting UNet
        ([3P] StableDiffusionXLInpaintPipeline with unet.config.in_channels == 9): every step's UNet input is the scaled
        latents followed by the mask and the masked-image latents (their CFG halves equal), and there is no blend.  It
        is required exactly when the UNet has 9 input channels.  It composes with begin_step, num_loop_steps and the
        other loop options, not with inpaint, start_step or stop_after (IHError).  The two tensors are copied once per
        call into a static buffer that the UNet's conv_in reads next to the step's latents (ops.im2col3x3_nchw_cat), so
        the step kernels are those of text-to-image.

        With an EulerAncestralDiscreteScheduler every option above works.  `generator` (a torch.Generator, a list of
        one per image, or None for the device's default generator) supplies the Gaussian noise of every step; before
        the steps run, the noise of exactly the steps this call executes is drawn from it, one draw per step in step
        order.  So `stop_after=k` followed by `start_step=k` with the same, continuing generator object reproduces the
        uninterrupted run.  The other schedulers draw nothing and ignore `generator`.

        `controlnet` = a ControlNetCall ([3P] StableDiffusionXLControlNetPipeline): at every step i with keep[i] = 1 the
        ControlNet runs on the step's model input (the CFG batch, or in guess mode with CFG the conditional half only)
        and its scaled residuals are added to the UNet's skip connections and mid-block output; at steps with keep[i] =
        0 the step is the plain one.  The control image's embedding is computed once per call.  It works with every
        scheduler and the loop options of text-to-image, not with begin_step, inpaint, unet_cond, start_step or
        stop_after (IHError).  It draws no random numbers.

        `controlnet` = a sequence of ControlNetCalls (up to 8, one per net, sharing guess_mode) is a Multi-ControlNet
        ([3P] MultiControlNetModel): at step i the nets with keep[i] = 1 run in net order and their scaled residuals
        are summed in fp16 and added in one launch.  diffusers runs an inactive net with scale 0; skipping it is exact
        (fp16(acc + 0) = acc).  A list of one call is the single-net case.

        `adapter` = an AdapterCall ([3P] StableDiffusionXLAdapterPipeline, T2I-Adapter): the call's 4 features are
        copied once into static buffers and its scale into a device fp32 value; at every step i with keep[i] = 1 the
        UNet adds them inside its encoder (UNet2DConditionModel.forward(adapter_residuals=)) to both CFG halves, at
        steps with keep[i] = 0 the step is the plain one.  There are at most two graphs per shape, with and without the
        features, and a new scale or image re-captures neither.  It works with every scheduler and the loop options
        of text-to-image, not with begin_step, inpaint, unet_cond, controlnet, start_step or stop_after (IHError).  It
        draws no random numbers."""
        use_cfg = guidance_scale > 1.0                                            # :223
        is_dpm = isinstance(self.scheduler, DPMSolverMultistepScheduler)         # the one scheduler dispatch
        is_ancestral = isinstance(self.scheduler, EulerAncestralDiscreteScheduler)
        ucfg = self.unet.config
        n, _, h, w = latents.shape
        L, T = prompt_embeds.shape[1], num_inference_steps
        # ---- every refusal comes before any allocation, copy or launch
        if use_cfg and (negative_prompt_embeds is None or negative_pooled is None):
            raise IHError("classifier-free guidance needs negative_prompt_embeds / negative_pooled")
        given = {"DPMSolverMultistepScheduler": is_dpm, "begin_step": bool(begin_step), "inpaint": inpaint is not None,
                 "unet_cond": unet_cond is not None, "controlnet": controlnet is not None,
                 "start_step": bool(start_step), "stop_after": stop_after is not None, "adapter": adapter is not None}
        for option, excluded, why in _EXCLUDES:
            clash = [o for o in excluded if given[o]]
            if given[option] and clash:
                raise IHError(f"{option} cannot be combined with {', '.join(clash)}: {why}")
        if (unet_cond is not None) != (ucfg.in_channels != ucfg.out_channels):
            raise IHError(f"unet_cond (mask, masked_image_latents) is required exactly for the 9-channel inpainting "
                          f"UNet; this UNet has {ucfg.in_channels} input channels")
        require_latent_size(ucfg, h, w)
        if is_ancestral and isinstance(generator, list) and len(generator) != n:
            raise IHError(f"got {len(generator)} generators for a batch of {n}")
        loop_T = T if num_loop_steps is None else int(num_loop_steps)
        if not 0 < loop_T <= T:
            raise IHError(f"num_loop_steps {num_loop_steps} outside the {T}-step schedule")
        if not 0 <= start_step <= loop_T:
            raise IHError(f"start_step {start_step} outside the {loop_T}-step loop")
        if begin_step and not 0 < begin_step < loop_T:
            raise IHError(f"begin_step {begin_step} leaves no step of the {loop_T}-step loop")
        if inpaint is not None:
            for name, t, want in zip(("image_latents", "noise", "mask"), inpaint,
                                     ((n, 4, h, w), (n, 4, h, w), (n, 1, h, w))):
                if tuple(t.shape) != want:
                    raise IHError(f"inpaint {name}: expected shape {want}, got {tuple(t.shape)}")
        if unet_cond is not None:
            want = ((n, 1, h, w), (n, ucfg.in_channels - ucfg.out_channels - 1, h, w))
            if tuple(tuple(t.shape) for t in unet_cond) != want:
                raise IHError(f"unet_cond: expected mask {want[0]} and masked_image_latents {want[1]}, got "
                              f"{tuple(unet_cond[0].shape)} and {tuple(unet_cond[1].shape)}")
        calls, keeps = [], []                   # per ControlNet: its call and keep list
        if controlnet is not None:
            calls = list(controlnet) if isinstance(controlnet, (list, tuple)) else [controlnet]
            if not 1 <= len(calls) <= IH_CN_MAX_NETS:
                raise IHError(f"controlnet: {len(calls)} ControlNetCalls, expected 1 .. {IH_CN_MAX_NETS}")
            if any(bool(c.guess_mode) != bool(calls[0].guess_mode) for c in calls):
                raise IHError("controlnet: all ControlNetCalls must share guess_mode")
            for j, call in enumerate(calls):
                mcfg = call.model.config
                if mcfg.block_out_channels != ucfg.block_out_channels:
                    raise IHError(f"ControlNet {j}: its block_out_channels differ from the UNet's")
                keeps.append([1.0] * T if call.keep is None else [float(k) for k in call.keep])
                if len(keeps[j]) != T:
                    raise IHError(f"ControlNet {j}: keep has {len(keeps[j])} entries for a {T}-step schedule")
                if tuple(call.image.shape) != (n, mcfg.conditioning_channels, 8 * h, 8 * w):
                    raise IHError(f"ControlNet {j}: image: expected {(n, mcfg.conditioning_channels, 8 * h, 8 * w)}, "
                                  f"got {tuple(call.image.shape)}")
        ad_keep = None
        if adapter is not None:
            if ucfg.in_channels != 4:
                raise IHError(f"adapter: the T2I-Adapter runs with the 4-channel UNet only (this one has "
                              f"{ucfg.in_channels} input channels)")
            feats = list(adapter.features)
            require_adapter_shapes(ucfg, h, w, [tuple(f.shape[1:]) for f in feats])
            if any(f.shape[0] != n for f in feats):
                raise IHError(f"adapter: features of {[f.shape[0] for f in feats]} images for a batch of {n}")
            ad_keep = [1.0] * T if adapter.keep is None else [float(k) for k in adapter.keep]
            if len(ad_keep) != T:
                raise IHError(f"adapter: keep has {len(ad_keep)} entries for a {T}-step schedule")
        start_step = begin_step or start_step
        steps = loop_T if stop_after is None else min(stop_after, loop_T)

        # ---- the loop record; inputs -> static device buffers (H2D copies when the caller hands over pinned tensors)
        timesteps, sigmas, _, coeffs = self._schedule(T)
        rescale = float(guidance_rescale or 0.0) if use_cfg else 0.0              # :352 needs CFG
        st = self._buffers(n, h, w, L, use_cfg)
        loop = _Loop(st, timesteps, sigmas, float(guidance_scale), use_cfg, rescale, (n, h, w, L, T),
                     self.scheduler.kind)
        neg_tid = time_ids if negative_time_ids is None else negative_time_ids
        if use_cfg:
            st["ehs"][:n].copy_(negative_prompt_embeds, non_blocking=True)    # CFG order [negative, positive], :296
            st["ehs"][n:].copy_(prompt_embeds, non_blocking=True)
            st["text_embeds"][:n].copy_(negative_pooled, non_blocking=True)
            st["text_embeds"][n:].copy_(pooled, non_blocking=True)
            st["time_ids"][:n].copy_(neg_tid, non_blocking=True)              # :298
            st["time_ids"][n:].copy_(time_ids, non_blocking=True)
        else:
            st["ehs"].copy_(prompt_embeds, non_blocking=True)
            st["text_embeds"].copy_(pooled, non_blocking=True)
            st["time_ids"].copy_(time_ids, non_blocking=True)
        C = ucfg.out_channels
        if is_dpm:      # the previous step's data prediction and the schedule index the loop starts at (first order)
            loop.coeffs = coeffs
            loop.dpm = {"prev_x0": self._buf("prev_x0", (n, h, w), (n, C, h, w)),
                        "loop_begin": self._buf("loop_begin", (n, h, w), (1,), torch.int32, zero=True)}
            loop.dpm["loop_begin"].fill_(start_step)
        elif is_ancestral:
            loop.coeffs = coeffs
            loop.noise = self._buf("step_noise", (n, h, w, T), (T, n, C, h, w), zero=True)
        if inpaint is not None:
            loop.ib = {name: self._buf(name, (n, h, w), t.shape) for name, t in
                       zip(("image_latents", "noise", "mask"), inpaint)}
            for name, t in zip(("image_latents", "noise", "mask"), inpaint):
                loop.ib[name].copy_(t, non_blocking=True)
            loop.ib["blend_end"] = self._buf("blend_end", (n, h, w), (1,), torch.int32, zero=True)
            loop.ib["blend_end"].fill_(loop_T)
        if unet_cond is not None:
            cond = loop.cond = self._buf("unet_cond", (n, h, w, use_cfg),
                                         (2 * n if use_cfg else n, ucfg.in_channels - C, h, w))
            for half in ((0, n), (n, 2 * n)) if use_cfg else ((0, n),):     # [3P] cat([mask] * 2) under CFG
                cond[half[0]:half[1], :1].copy_(unet_cond[0], non_blocking=True)
                cond[half[0]:half[1], 1:].copy_(unet_cond[1], non_blocking=True)
        if adapter is not None:     # the features of one CFG half; the UNet adds them to each half
            bufs = [self._buf("adapter_feature", (k, n, h, w), tuple(f.shape)) for k, f in enumerate(adapter.features)]
            for b, f in zip(bufs, adapter.features):
                b.copy_(f, non_blocking=True)
            scale = self._buf("adapter_scale", (n, h, w), (2,), torch.float32, zero=True)
            scale.fill_(float(adapter.scale))
            loop.adapter = (bufs, scale)
        self.unet.prepare_conditioning(st["ehs"], st["text_embeds"], st["time_ids"])
        nets = []                               # per ControlNet: (model, conditioning embedding, scale vector)
        b_cn0 = n if (use_cfg and calls and calls[0].guess_mode) else 0      # guess mode + CFG: the conditional half
        b_cn = (2 * n if use_cfg else n) - b_cn0
        for j, call in enumerate(calls):
            model = call.model
            emb = self._buf("cn_emb", (j, b_cn, h, w), (b_cn, h, w, ucfg.block_out_channels[0]))
            scale = self._buf("cn_scale", (j, b_cn, h, w), (10,), torch.float32, zero=True)
            model.embed_condition(call.image.to(self.device, torch.float16).contiguous(), out=emb[:n])
            if b_cn > n:                                        # [3P] cat([image] * 2) under CFG
                emb[n:].copy_(emb[:n])
            scale.copy_(controlnet_scales(call.conditioning_scale, bool(call.guess_mode)))
            model.prepare_conditioning(st["ehs"][b_cn0:], st["text_embeds"][b_cn0:], st["time_ids"][b_cn0:])
            nets.append((model, emb, scale))
        self._restart(loop, latents, start_step)                                       # :332-334
        self._loop = loop

        b0, n_loop = begin_step, loop_T - begin_step                         # the (truncated) list the loop sees

        def scale_at(i: int) -> float:
            off = ((i - b0) / n_loop < control_guidance_start) or ((i - b0 + 1) / n_loop > control_guidance_end)  # :326-329
            return 0.0 if off else float(ip_scale)

        def cn_at(i: int):
            # the nets with keep[i] = 1, in net order; diffusers runs the others at scale 0, which adds exactly nothing
            active = tuple(j for j, keep in enumerate(keeps) if keep[i] > 0)
            return (active, [nets[j] for j in active], b_cn0) if active else None

        def ad_at(i: int) -> bool:
            return ad_keep is not None and ad_keep[i] > 0

        if self.use_cuda_graph:
            if self._epoch != getattr(self.unet, "graph_epoch", 0):       # weights / processors changed since capture
                self._graphs.clear()
                self._epoch = getattr(self.unet, "graph_epoch", 0)
            for j, (model, _, _) in enumerate(nets):
                seen = self._cn_epochs.get(j)
                if seen is None or seen[0] is not model or seen[1] != model.graph_epoch:   # another / a reloaded net
                    self._graphs = {k: v for k, v in self._graphs.items() if k.controlnet is None or j not in k.controlnet[2]}
                    self._cn_epochs[j] = (model, model.graph_epoch)
            needed = {}
            for i in range(start_step, steps):
                needed.setdefault(loop.graph_key(scale_at(i), cn_at(i), ad_at(i)), (scale_at(i), cn_at(i), ad_at(i)))
            captured = False
            for _ in range(4):      # a warm-up may grow a scratch buffer, which invalidates graphs captured before it
                gen = ops.workspace_generation()
                missing = [k for k in needed if self._graphs.get(k, (None, -1))[1] != gen]
                if not missing:
                    break
                for k in missing:
                    sc, cn_step, ad_step = needed[k]
                    self.set_scale(sc)
                    self._graphs[k] = (self._capture(loop, cn_step, ad_step), ops.workspace_generation())
                    captured = True
            else:
                raise IHError("scratch buffers kept growing during graph capture")
            if captured:            # the warm-up pass of a capture advances the state once
                self._restart(loop, latents, start_step)
        if loop.noise is not None:
            self._draw_ancestral_noise(loop.noise, generator, start_step, steps)
        for i in range(start_step, steps):
            sc = scale_at(i)
            if self.use_cuda_graph:
                self._graphs[loop.graph_key(sc, cn_at(i), ad_at(i))][0].replay()
            else:
                self.set_scale(sc)
                self._step(loop, cn_at(i), ad_at(i))
            if callback is not None and (i - b0) % callback_steps == 0:           # :359-363 (Euler: order 1, no warm-up)
                callback(i - b0, timesteps[i], st["latents"])
        self.set_scale(ip_scale)
        return st["latents"].clone()

    def _capture(self, loop: _Loop, cn=None, adapter: bool = False):
        # warm-up on a side stream (sets kernel attributes, fills the TMA descriptor cache, sizes the allocator and
        # the library's scratch buffers)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            loop.st["step"].zero_()
            self._step(loop, cn, adapter)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        loop.st["step"].zero_()
        g = torch.cuda.CUDAGraph()
        before = ops.launch_count()
        with torch.cuda.graph(g):
            self._step(loop, cn, adapter)
        self.last_launches_per_step = ops.launch_count() - before
        self.graphs_captured += 1
        return g
