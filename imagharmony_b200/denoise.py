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

Graph lifetime: a captured graph holds raw pointers.  Everything it reads lives in buffers that are owned per shape
and never freed while the graph exists -- the engine's static inputs (`_static`, `_inpaint_static`, `_dpm_static`,
`_cond_static`, `_ancestral_noise`, `_cn_static`: each ControlNet's conditioning embedding and scale vector), the schedule tables (`_tables`, `_coeffs`), the processors'
K/V buffers and the UNet's add-embedding buffer (per-shape dicts inside those objects), and the library's grow-only
scratch buffers whose re-allocation bumps `ops.workspace_generation()`.  A graph is replayed only if it was captured
under the current UNet `graph_epoch` (weights / processors unchanged) and the current workspace generation; otherwise
it is re-captured; a graph with ControlNets also needs each of its nets to be the object, at the `graph_epoch`, it was
captured with (tracked per net index, so reloading one net re-captures only the graphs that contain it).

ControlNet (`run(controlnet=...)`): a step runs the active ControlNets' forwards in net order, then the UNet with
their residuals summed and injected after the mid block in one launch, then the unchanged step kernel, all in the one
graph.  There is one graph per distinct set of active nets (staggered windows of K nets give at most 2K + 1); steps
where no net is active (keep[i] = 0 for all) replay the ControlNet-free graph.  The scale vectors are read from device
memory, so a new controlnet_conditioning_scale does not re-capture.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import ops
from ._lib import IH_CN_MAX_NETS, IHError
from .controlnet import controlnet_scales
from .scheduler import DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler, EulerDiscreteScheduler
from .unet import UNet2DConditionModel


class DenoiseEngine:
    def __init__(self, unet: UNet2DConditionModel, use_cuda_graph: bool = True,
                 scheduler: Optional[Union[EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                                           DPMSolverMultistepScheduler]] = None):
        self.unet = unet
        self.device = unet.conv_in.weight.device
        self.scheduler = scheduler or EulerDiscreteScheduler()      # the pipeline's own scheduler object when given
        self.use_cuda_graph = use_cuda_graph and self.device.type == "cuda"
        self._graphs: Dict[Tuple, Tuple[torch.cuda.CUDAGraph, int]] = {}   # key -> (graph, workspace generation)
        self._static: Dict[Tuple, dict] = {}
        self._inpaint_static: Dict[Tuple, dict] = {}
        self._dpm_static: Dict[Tuple, dict] = {}
        self._cond_static: Dict[Tuple, torch.Tensor] = {}               # 9-channel UNet: mask | masked-image latents
        self._tables: Dict[Tuple[str, int], Tuple[torch.Tensor, torch.Tensor, float]] = {}
        self._coeffs: Dict[Tuple[str, int], torch.Tensor] = {}         # DPM-Solver++ / Euler Ancestral coefficients
        self._ancestral_noise: Dict[Tuple[int, int, int, int], torch.Tensor] = {}   # Euler Ancestral step noise
        # ControlNet: conditioning embedding + scale vector per (net index, shape)
        self._cn_static: Dict[Tuple, dict] = {}
        # net index -> (ControlNet, graph_epoch) the graphs with that net were captured for.  The model object itself is
        # kept, not its id: a freed model's id can be reused by a new one that reaches the same epoch
        self._cn_epochs: Dict[int, Tuple] = {}
        self._epoch = getattr(unet, "graph_epoch", 0)
        self.last_launches_per_step = 0
        self.graphs_captured = 0

    # ------------------------------------------------------------------------------------------------------------
    def tables(self, num_steps: int):
        """(timesteps fp32, sigmas fp32, init_noise_sigma) of the engine's scheduler on the device, per (kind, T);
        with DPM-Solver++ and Euler Ancestral the coefficient table is kept next to them (`coeffs`)."""
        key = (self.scheduler.kind, num_steps)
        t = self._tables.get(key)
        if t is None:
            s = self.scheduler.set_timesteps(num_steps)
            t = (torch.from_numpy(s.timesteps.astype(np.float32)).to(self.device),
                 torch.from_numpy(s.sigmas).to(self.device), s.init_noise_sigma)
            self._tables[key] = t
            if isinstance(self.scheduler, (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler)):
                self._coeffs[key] = torch.from_numpy(s.coeffs).to(self.device)
        return t

    def coeffs(self, num_steps: int) -> torch.Tensor:
        self.tables(num_steps)
        return self._coeffs[(self.scheduler.kind, num_steps)]

    def set_scale(self, scale: float) -> None:
        """IPAdapter.set_scale / pipeline.set_scale (ip_adapter.py:179-182, custom_pipelines.py:17-20)."""
        for p in self.unet.attn_processors.values():
            if hasattr(p, "to_k_ip"):
                p.scale = scale

    def invalidate_graphs(self) -> None:
        self._graphs.clear()

    def _buffers(self, n: int, h: int, w: int, L: int, use_cfg: bool = True):
        key = (n, h, w, L, use_cfg)
        st = self._static.get(key)
        if st is None:
            cfg = self.unet.config
            dev = self.device
            b = 2 * n if use_cfg else n
            st = {
                "latents": torch.empty((n, cfg.out_channels, h, w), dtype=torch.float16, device=dev),
                "model_in": torch.empty((b, cfg.out_channels, h, w), dtype=torch.float16, device=dev),
                "ehs": torch.empty((b, L, cfg.cross_attention_dim), dtype=torch.float16, device=dev),
                "text_embeds": torch.empty((b, cfg.pooled_embed_dim), dtype=torch.float16, device=dev),
                "time_ids": torch.empty((b, 6), dtype=torch.float32, device=dev),
                "step": torch.zeros((1,), dtype=torch.int32, device=dev),
            }
            self._static[key] = st
        return st

    def _inpaint_buffers(self, n: int, h: int, w: int):
        """Static inputs of the inpainting step, per (n, h, w) and never freed (the graph-lifetime rule above)."""
        key = (n, h, w)
        ib = self._inpaint_static.get(key)
        if ib is None:
            dev = self.device
            ib = {"image_latents": torch.empty((n, 4, h, w), dtype=torch.float16, device=dev),
                  "noise": torch.empty((n, 4, h, w), dtype=torch.float16, device=dev),
                  "mask": torch.empty((n, 1, h, w), dtype=torch.float16, device=dev),
                  "blend_end": torch.zeros((1,), dtype=torch.int32, device=dev)}
            self._inpaint_static[key] = ib
        return ib

    def _dpm_buffers(self, n: int, h: int, w: int):
        """DPM-Solver++ state per (n, h, w), never freed (the graph-lifetime rule above): the previous step's data
        prediction and the schedule index the loop starts at (its step is first order)."""
        key = (n, h, w)
        db = self._dpm_static.get(key)
        if db is None:
            dev = self.device
            db = {"prev_x0": torch.empty((n, self.unet.config.out_channels, h, w), dtype=torch.float16, device=dev),
                  "loop_begin": torch.zeros((1,), dtype=torch.int32, device=dev)}
            self._dpm_static[key] = db
        return db

    def _ancestral_buffer(self, n: int, h: int, w: int, T: int) -> torch.Tensor:
        """Euler Ancestral step noise [T, n, C, h, w] per (n, h, w, T), never freed (the graph-lifetime rule above).
        Zero-filled, so that a capture's warm-up step reads finite values."""
        key = (n, h, w, T)
        buf = self._ancestral_noise.get(key)
        if buf is None:
            buf = torch.zeros((T, n, self.unet.config.out_channels, h, w), dtype=torch.float16, device=self.device)
            self._ancestral_noise[key] = buf
        return buf

    def _cond_buffer(self, n: int, h: int, w: int, use_cfg: bool) -> torch.Tensor:
        """The 9-channel UNet's extra input [b, C_in - C_lat, h, w] (mask | masked-image latents, both CFG halves) per
        (n, h, w, use_cfg), never freed (the graph-lifetime rule above)."""
        key = (n, h, w, use_cfg)
        buf = self._cond_static.get(key)
        if buf is None:
            cfg = self.unet.config
            buf = torch.empty((2 * n if use_cfg else n, cfg.in_channels - cfg.out_channels, h, w), dtype=torch.float16,
                              device=self.device)
            self._cond_static[key] = buf
        return buf

    def _cn_buffers(self, net: int, b: int, h: int, w: int) -> dict:
        """ControlNet static inputs per (net index, ControlNet batch, h, w), never freed (the graph-lifetime rule above):
        the conditioning embedding NHWC [b, h, w, C0] and the fp32 scale vector [10], refilled by every call."""
        key = (net, b, h, w)
        cb = self._cn_static.get(key)
        if cb is None:
            C0 = self.unet.config.block_out_channels[0]
            cb = {"emb": torch.empty((b, h, w, C0), dtype=torch.float16, device=self.device),
                  "scale": torch.zeros((10,), dtype=torch.float32, device=self.device)}
            self._cn_static[key] = cb
        return cb

    def _draw_ancestral_noise(self, buf: torch.Tensor, generator, begin: int, end: int) -> None:
        """Rows [begin, end) of the step noise, one draw per step in step order, as [3P] diffusers' randn_tensor draws
        it inside EulerAncestralDiscreteScheduler.step: fp16, shaped like the guided prediction, on the generator's
        device (a CPU generator draws on the CPU), one [1, C, h, w] draw per generator of a list, and from the device's
        default generator when `generator` is None."""
        shape = tuple(buf.shape[1:])
        for i in range(begin, end):
            if isinstance(generator, list):
                row = torch.cat([torch.randn((1,) + shape[1:], generator=g, device=g.device, dtype=torch.float16)
                                 .to(self.device) for g in generator])
            else:
                dev = generator.device if generator is not None else self.device
                row = torch.randn(shape, generator=generator, device=dev, dtype=torch.float16)
            buf[i].copy_(row)

    def _first_input(self, st, sigmas, use_cfg: bool, dpm, anc=None) -> None:
        """The UNet input of the loop's first step from st["latents"] (custom_pipelines.py:332-334)."""
        if anc is not None:      # the convention of the ancestral kernel's later inputs: x * fp32(1 / sqrt(s^2 + 1))
            ops.euler_ancestral_scale_input(st["latents"], st["model_in"], anc[0], st["step"], duplicate=use_cfg)
            return
        if dpm is None:
            ops.scale_model_input(st["latents"], st["model_in"], sigmas, st["step"], duplicate=use_cfg)
            return
        n = st["latents"].shape[0]                   # DPM-Solver++: scale_model_input is the identity
        st["model_in"][:n].copy_(st["latents"])
        if use_cfg:
            st["model_in"][n:].copy_(st["latents"])

    def _step(self, st, timesteps, sigmas, guidance, use_cfg=True, rescale=0.0, ib=None, dpm=None, anc=None, cond=None,
              cn=None):
        residuals = None
        if cn is not None:          # (active net indices, [(ControlNet, static buffers)], first image they run on)
            _, nets, b0 = cn
            outs = [model(st["model_in"][b0:], timesteps, st["ehs"][b0:], text_embeds=st["text_embeds"][b0:],
                          time_ids=st["time_ids"][b0:], step=st["step"], cond_embedding=cb["emb"], scale=cb["scale"])
                    for model, cb in nets]
            residuals = (outs[0] if len(outs) == 1 else outs, b0)
        noise = self.unet(st["model_in"], timesteps, st["ehs"], st["text_embeds"], st["time_ids"], step=st["step"],
                          cond=cond, controlnet_residuals=residuals)
        if dpm is not None:
            db, coeffs = dpm
            ops.dpm_solver_step(noise, st["latents"], st["model_in"], db["prev_x0"], coeffs, st["step"],
                                db["loop_begin"], guidance, use_cfg=use_cfg, guidance_rescale=rescale)
        elif anc is not None:
            blend = None if ib is None else (ib["image_latents"], ib["noise"], ib["mask"], ib["blend_end"])
            ops.euler_ancestral_step(noise, st["latents"], st["model_in"], anc[0], anc[1], st["step"], guidance,
                                     use_cfg=use_cfg, guidance_rescale=rescale, inpaint=blend)
        elif ib is None:
            ops.euler_step(noise, st["latents"], st["model_in"], sigmas, st["step"], guidance, use_cfg=use_cfg,
                           guidance_rescale=rescale)
        else:
            ops.euler_inpaint_step(noise, st["latents"], st["model_in"], sigmas, st["step"], guidance,
                                   ib["image_latents"], ib["noise"], ib["mask"], ib["blend_end"], use_cfg=use_cfg,
                                   guidance_rescale=rescale)

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
            unet_cond: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, controlnet=None) -> torch.Tensor:
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
        (fp16(acc + 0) = acc).  A list of one call is the single-net case."""
        use_cfg = guidance_scale > 1.0                                            # :223
        if use_cfg and (negative_prompt_embeds is None or negative_pooled is None):
            raise IHError("classifier-free guidance needs negative_prompt_embeds / negative_pooled")
        is_dpm = isinstance(self.scheduler, DPMSolverMultistepScheduler)         # the one scheduler dispatch
        is_ancestral = isinstance(self.scheduler, EulerAncestralDiscreteScheduler)
        if is_dpm and (begin_step or inpaint is not None or unet_cond is not None or start_step
                       or stop_after is not None):
            raise IHError("DPMSolverMultistepScheduler runs whole text-to-image loops: begin_step (image-to-image), "
                          "inpaint, unet_cond, start_step and stop_after need EulerDiscreteScheduler")
        ucfg = self.unet.config
        if (unet_cond is not None) != (ucfg.in_channels != ucfg.out_channels):
            raise IHError(f"unet_cond (mask, masked_image_latents) is required exactly for the 9-channel inpainting "
                          f"UNet; this UNet has {ucfg.in_channels} input channels")
        if unet_cond is not None and (inpaint is not None or start_step or stop_after is not None):
            raise IHError("unet_cond cannot be combined with inpaint / start_step / stop_after")
        if controlnet is not None and (begin_step or inpaint is not None or unet_cond is not None or start_step
                                       or stop_after is not None):
            raise IHError("controlnet runs text-to-image loops: it cannot be combined with begin_step, inpaint, "
                          "unet_cond, start_step or stop_after")
        n, _, h, w = latents.shape
        if is_ancestral and isinstance(generator, list) and len(generator) != n:
            raise IHError(f"got {len(generator)} generators for a batch of {n}")
        L = prompt_embeds.shape[1]
        T = num_inference_steps
        loop_T = T if num_loop_steps is None else int(num_loop_steps)
        if not 0 < loop_T <= T:
            raise IHError(f"num_loop_steps {num_loop_steps} outside the {T}-step schedule")
        rescale = float(guidance_rescale or 0.0) if use_cfg else 0.0              # :352 needs CFG
        timesteps, sigmas, _ = self.tables(T)
        st = self._buffers(n, h, w, L, use_cfg)
        # inputs -> static device buffers (H2D copies when the caller hands over pinned host tensors)
        st["latents"].copy_(latents, non_blocking=True)
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
        dpm = anc = None
        if is_dpm:
            dpm = (self._dpm_buffers(n, h, w), self.coeffs(T))
        elif is_ancestral:
            anc = (self.coeffs(T), self._ancestral_buffer(n, h, w, T))
        ib = None
        if inpaint is not None:
            if start_step or stop_after is not None:
                raise IHError("inpaint cannot be combined with start_step / stop_after")
            ib = self._inpaint_buffers(n, h, w)
            for name, t in zip(("image_latents", "noise", "mask"), inpaint):
                if tuple(t.shape) != tuple(ib[name].shape):
                    raise IHError(f"inpaint {name}: expected shape {tuple(ib[name].shape)}, got {tuple(t.shape)}")
                ib[name].copy_(t, non_blocking=True)
            ib["blend_end"].fill_(loop_T)
        cond = None
        if unet_cond is not None:
            cond = self._cond_buffer(n, h, w, use_cfg)
            mask, masked = unet_cond
            want = ((n, 1, h, w), (n, cond.shape[1] - 1, h, w))
            if (tuple(mask.shape), tuple(masked.shape)) != want:
                raise IHError(f"unet_cond: expected mask {want[0]} and masked_image_latents {want[1]}, got "
                              f"{tuple(mask.shape)} and {tuple(masked.shape)}")
            for half in ((0, n), (n, 2 * n)) if use_cfg else ((0, n),):     # [3P] cat([mask] * 2) under CFG
                cond[half[0]:half[1], :1].copy_(mask, non_blocking=True)
                cond[half[0]:half[1], 1:].copy_(masked, non_blocking=True)
        if not 0 <= start_step <= loop_T:
            raise IHError(f"start_step {start_step} outside the {loop_T}-step loop")
        if begin_step:
            if start_step or stop_after is not None:
                raise IHError("begin_step (image-to-image) cannot be combined with start_step / stop_after")
            if not 0 < begin_step < loop_T:
                raise IHError(f"begin_step {begin_step} leaves no step of the {loop_T}-step loop")
            start_step = begin_step
        st["step"].fill_(start_step)
        if dpm is not None:
            dpm[0]["loop_begin"].fill_(start_step)
        self.unet.prepare_conditioning(st["ehs"], st["text_embeds"], st["time_ids"])
        nets, keeps, b_cn0 = [], [], 0          # per ControlNet: (model, static buffers), keep list; first image
        if controlnet is not None:
            calls = list(controlnet) if isinstance(controlnet, (list, tuple)) else [controlnet]
            if not 1 <= len(calls) <= IH_CN_MAX_NETS:
                raise IHError(f"controlnet: {len(calls)} ControlNetCalls, expected 1 .. {IH_CN_MAX_NETS}")
            guess = bool(calls[0].guess_mode)
            if any(bool(c.guess_mode) != guess for c in calls):
                raise IHError("controlnet: all ControlNetCalls must share guess_mode")
            b_cn0 = n if (use_cfg and guess) else 0                 # guess mode + CFG: the conditional half only
            b_cn = (2 * n if use_cfg else n) - b_cn0
            for j, call in enumerate(calls):
                model = call.model
                if model.config.block_out_channels != ucfg.block_out_channels:
                    raise IHError(f"ControlNet {j}: its block_out_channels differ from the UNet's")
                keep = [1.0] * T if call.keep is None else [float(k) for k in call.keep]
                if len(keep) != T:
                    raise IHError(f"ControlNet {j}: keep has {len(keep)} entries for a {T}-step schedule")
                image = call.image
                if tuple(image.shape) != (n, model.config.conditioning_channels, 8 * h, 8 * w):
                    raise IHError(f"ControlNet {j}: image: expected "
                                  f"{(n, model.config.conditioning_channels, 8 * h, 8 * w)}, got {tuple(image.shape)}")
                cb = self._cn_buffers(j, b_cn, h, w)
                model.embed_condition(image.to(self.device, torch.float16).contiguous(), out=cb["emb"][:n])
                if b_cn > n:                                        # [3P] cat([image] * 2) under CFG
                    cb["emb"][n:].copy_(cb["emb"][:n])
                cb["scale"].copy_(controlnet_scales(call.conditioning_scale, guess))
                model.prepare_conditioning(st["ehs"][b_cn0:], st["text_embeds"][b_cn0:], st["time_ids"][b_cn0:])
                nets.append((model, cb))
                keeps.append(keep)
        self._first_input(st, sigmas, use_cfg, dpm, anc)                               # :332-334

        steps = loop_T if stop_after is None else min(stop_after, loop_T)

        b0, n_loop = begin_step, loop_T - begin_step                         # the (truncated) list the loop sees

        def scale_at(i: int) -> float:
            off = ((i - b0) / n_loop < control_guidance_start) or ((i - b0 + 1) / n_loop > control_guidance_end)  # :326-329
            return 0.0 if off else float(ip_scale)

        def cn_at(i: int):
            # the nets with keep[i] = 1, in net order; diffusers runs the others at scale 0, which adds exactly nothing
            active = tuple(j for j, keep in enumerate(keeps) if keep[i] > 0)
            return (active, [nets[j] for j in active], b_cn0) if active else None

        def gkey(scale: float, cn_step):
            return (n, h, w, L, T, use_cfg, float(guidance_scale), rescale, scale, self.scheduler.kind, cond is not None,
                    ib is not None, None if cn_step is None else ("controlnet", cn_step[2] > 0, cn_step[0]))

        if self.use_cuda_graph:
            if self._epoch != getattr(self.unet, "graph_epoch", 0):       # weights / processors changed since capture
                self._graphs.clear()
                self._epoch = getattr(self.unet, "graph_epoch", 0)
            for j, (model, _) in enumerate(nets):
                seen = self._cn_epochs.get(j)
                if seen is None or seen[0] is not model or seen[1] != model.graph_epoch:   # another / a reloaded net
                    self._graphs = {k: v for k, v in self._graphs.items() if k[-1] is None or j not in k[-1][2]}
                    self._cn_epochs[j] = (model, model.graph_epoch)
            needed = {}
            for i in range(start_step, steps):
                needed.setdefault(gkey(scale_at(i), cn_at(i)), (scale_at(i), cn_at(i)))
            captured = False
            for _ in range(4):      # a warm-up may grow a scratch buffer, which invalidates graphs captured before it
                gen = ops.workspace_generation()
                missing = [k for k in needed if self._graphs.get(k, (None, -1))[1] != gen]
                if not missing:
                    break
                for k in missing:
                    sc, cn_step = needed[k]
                    self.set_scale(sc)
                    g = self._capture(st, timesteps, sigmas, guidance_scale, use_cfg, rescale, ib, dpm, anc, cond,
                                      cn_step)
                    self._graphs[k] = (g, ops.workspace_generation())
                    captured = True
            else:
                raise IHError("scratch buffers kept growing during graph capture")
            if captured:
                # the warm-up pass of a capture advances the state once: restore the initial state
                st["latents"].copy_(latents, non_blocking=True)
                st["step"].fill_(start_step)
                self._first_input(st, sigmas, use_cfg, dpm, anc)
        if anc is not None:
            self._draw_ancestral_noise(anc[1], generator, start_step, steps)
        for i in range(start_step, steps):
            sc = scale_at(i)
            if self.use_cuda_graph:
                self._graphs[gkey(sc, cn_at(i))][0].replay()
            else:
                self.set_scale(sc)
                self._step(st, timesteps, sigmas, guidance_scale, use_cfg, rescale, ib, dpm, anc, cond, cn_at(i))
            if callback is not None and (i - b0) % callback_steps == 0:           # :359-363 (Euler: order 1, no warm-up)
                callback(i - b0, timesteps[i], st["latents"])
        self.set_scale(ip_scale)
        return st["latents"].clone()

    def _capture(self, st, timesteps, sigmas, guidance, use_cfg=True, rescale=0.0, ib=None, dpm=None, anc=None,
                 cond=None, cn=None):
        # warm-up on a side stream (sets kernel attributes, fills the TMA descriptor cache, sizes the allocator and
        # the library's scratch buffers)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            st["step"].zero_()
            self._step(st, timesteps, sigmas, guidance, use_cfg, rescale, ib, dpm, anc, cond, cn)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        st["step"].zero_()
        g = torch.cuda.CUDAGraph()
        before = ops.launch_count()
        with torch.cuda.graph(g):
            self._step(st, timesteps, sigmas, guidance, use_cfg, rescale, ib, dpm, anc, cond, cn)
        self.last_launches_per_step = ops.launch_count() - before
        self.graphs_captured += 1
        return g
