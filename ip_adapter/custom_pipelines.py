"""StableDiffusionXLCustomPipeline with the reference's call surface (ip_adapter/custom_pipelines.py:16-394) on the
native UNet / DenoiseEngine.  The reference class derives from diffusers' StableDiffusionXLPipeline; diffusers is not
a dependency here, so the pieces the reference touches are provided directly:

    .unet (.config.{cross_attention_dim, block_out_channels, in_channels}, .attn_processors, .set_attn_processor)
    .scheduler, .set_scale(scale), .to(device), .enable_vae_tiling(), .encode_prompt(...), .__call__(...)

Denoise loop semantics follow custom_pipelines.py:188-363 (CFG batch [negative, positive], per-step IP-scale gating
by control_guidance_start/end, Euler update); the loop itself runs as replayed CUDA graphs (imagharmony_b200/denoise.py).
Text-to-image also runs DPM-Solver++ 2M: pass `scheduler=DPMSolverMultistepScheduler.from_config(pipe.scheduler.config,
use_karras_sigmas=True)` or assign it to `pipe.scheduler`, as with diffusers, and UniPC likewise:
`pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)`.  Text-to-image, image-to-image and
inpainting run Euler Ancestral (`EulerAncestralDiscreteScheduler.from_config(pipe.scheduler.config)`), whose per-step
noise comes from the call's `generator` in diffusers' order.
VAE decode / PIL post-processing (:365-386, scope row f1) runs on the native decoder `imagharmony_b200.vae` when the
pipeline owns one (`from_random`, or `from_pretrained` with a `vae/` folder); a `vae_decode` callable overrides it and
`output_type="latent"` skips it.  `pipe.vae = AutoencoderTiny.from_pretrained(dir)` swaps in the native tiny decoder
(imagharmony_b200.taesd, TAESD-XL); image-to-image and inpainting then refuse to encode a pixel image.
"""
from __future__ import annotations

import dataclasses
import hashlib
import json
import os
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch

from imagharmony_b200 import ops
from imagharmony_b200._lib import IHError
from imagharmony_b200.config import SDXL_BASE, SDXL_CONTROLNET, ControlNetConfig, UNetConfig, config_from_diffusers
from imagharmony_b200.denoise import DenoiseEngine
from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                        EulerDiscreteScheduler, UniPCMultistepScheduler, randn_tensor)
from imagharmony_b200.unet import UNet2DConditionModel, require_latent_size
from imagharmony_b200.weights import random_module

from .utils import is_torch2_available

if is_torch2_available():
    from .attention_processor import IPAttnProcessor2_0 as IPAttnProcessor
else:  # pragma: no cover
    from .attention_processor import IPAttnProcessor


@dataclass
class StableDiffusionXLPipelineOutput:
    images: Any


class SyntheticPromptEncoder:
    """Stand-in for the two CLIP text encoders when no weights are on disk (this environment has no network):
    deterministic N(0,1) embeddings seeded by a hash of the prompt string.  Shapes/dtypes match encode_prompt [3P]."""

    def __init__(self, cfg: UNetConfig):
        self.cfg = cfg

    def __call__(self, prompts: List[str]) -> Tuple[torch.Tensor, torch.Tensor]:
        hs, pooled = [], []
        for p in prompts:
            seed = int.from_bytes(hashlib.sha256(p.encode()).digest()[:8], "little") & 0x7FFFFFFFFFFFFFFF
            g = torch.Generator("cpu").manual_seed(seed)
            hs.append(torch.randn(77, self.cfg.cross_attention_dim, generator=g))
            pooled.append(torch.randn(self.cfg.pooled_embed_dim, generator=g))
        return torch.stack(hs).half(), torch.stack(pooled).half()


def _fraction(value) -> bool:
    """[3P] diffusers' denoising_value_valid: denoising_start / denoising_end take effect only as a float in (0, 1)."""
    return isinstance(value, float) and 0 < value < 1


def _denoising_cutoff(num_train_timesteps: int, fraction: float) -> int:
    """[3P] The timestep that a valid denoising_start / denoising_end splits the schedule at."""
    return int(round(num_train_timesteps - fraction * num_train_timesteps))


def denoising_start_begin_step(timesteps, num_train_timesteps: int, denoising_start: float) -> int:
    """[3P] StableDiffusionXLImg2ImgPipeline.get_timesteps with a valid `denoising_start` (first-order schedulers): the
    loop runs the n timesteps below the cutoff (_denoising_cutoff), the last n of the schedule, so it begins at
    index len(timesteps) - n.  A base run with denoising_end = denoising_start keeps the timesteps at or above the same
    cutoff, so it ends at that same index: the handoff repeats and skips no step."""
    cutoff = _denoising_cutoff(num_train_timesteps, denoising_start)
    return len(timesteps) - int(sum(1 for t in timesteps if t < cutoff))


def _read_json(path: str, *parts: str) -> dict:
    f = os.path.join(path, *parts)
    if not os.path.exists(f):
        return {}
    with open(f) as fh:
        return json.load(fh)


@dataclass
class _Pretrained:
    """The parts of an SDXL folder that from_pretrained builds a pipeline from."""
    unet: UNet2DConditionModel
    prompt_encoder: Optional[Callable]      # ClipPromptEncoder, None without text encoders on disk
    vae: Any                                # AutoencoderKLDecoder, None without a vae/ folder
    vae_state: Optional[Dict[str, torch.Tensor]]
    vae_config: Any
    index: dict                             # model_index.json, {} without one


def _pil_list(image) -> Optional[list]:
    """A PIL image or a non-empty list / tuple of them as a list; None for anything else."""
    from PIL import Image
    if isinstance(image, Image.Image):
        return [image]
    if isinstance(image, (list, tuple)) and image and isinstance(image[0], Image.Image):
        return list(image)
    return None


def _load_images(image, size: Callable[[int, int], Tuple[int, int]], what: str, vae_scale_factor: int) -> torch.Tensor:
    """PIL image(s) -> RGB, Lanczos resize, / 255; a [B, 3, H, W] / [3, H, W] tensor -> float, nearest resize; both to
    the (height, width) that `size` gives for the first image's (H, W).  -> float32 [B, 3, height, width], PIL images
    in [0, 1], a tensor in its own range.  `what` names the image in the error messages."""
    import numpy as np
    from PIL import Image
    images = _pil_list(image)
    if images is not None:
        w0, h0 = images[0].size
        h, w = size(h0, w0)
        if h <= 0 or w <= 0:
            raise ValueError(f"{what} of size {images[0].size} is smaller than {vae_scale_factor} pixels")
        images = [im.convert("RGB") if im.mode != "RGB" else im for im in images]
        images = [im if im.size == (w, h) else im.resize((w, h), resample=Image.LANCZOS) for im in images]
        arr = np.stack([np.array(im).astype(np.float32) / 255.0 for im in images])
        return torch.from_numpy(arr).permute(0, 3, 1, 2).contiguous()
    if isinstance(image, torch.Tensor):
        x = image.unsqueeze(0) if image.dim() == 3 else image
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"{what} tensor must be [B, 3, H, W] or [3, H, W], got {tuple(image.shape)}")
        x = x.float()
        h, w = size(x.shape[2], x.shape[3])
        if h <= 0 or w <= 0:
            raise ValueError(f"{what} of size {tuple(x.shape[2:])} is smaller than {vae_scale_factor} pixels")
        if (h, w) != tuple(x.shape[2:]):
            x = torch.nn.functional.interpolate(x, size=(h, w))
        return x.contiguous()
    raise ValueError(f"`image` must be a PIL image, a list of them or a tensor, got {type(image).__name__}")


class StableDiffusionXLCustomPipeline:
    vae_scale_factor = 8
    force_zeros_for_empty_prompt = True     # [3P] SDXL-base pipeline config; from_pretrained reads model_index.json
    TIME_IDS = (6,)                         # the UNet micro-conditioning id counts this pipeline forms

    def __init__(self, unet: UNet2DConditionModel, prompt_encoder: Optional[Callable] = None,
                 vae_decode: Optional[Callable] = None,
                 scheduler: Optional[Union[EulerDiscreteScheduler, DPMSolverMultistepScheduler,
                                            UniPCMultistepScheduler]] = None, vae=None):
        if unet.config.num_time_ids not in self.TIME_IDS:
            raise IHError(f"{type(self).__name__} needs a UNet with {' or '.join(map(str, self.TIME_IDS))} "
                          f"micro-conditioning ids; this one has {unet.config.num_time_ids} (a UNet that requires an "
                          "aesthetics score, the SDXL refiner, runs in StableDiffusionXLImg2ImgPipeline)")
        self.unet = unet
        self.vae = vae                      # imagharmony_b200.vae.AutoencoderKLDecoder, taesd.AutoencoderTiny or None
        self.scheduler = scheduler or EulerDiscreteScheduler()
        self.prompt_encoder = prompt_encoder or SyntheticPromptEncoder(unet.config)
        self.vae_decode = vae_decode
        self.default_sample_size = unet.config.sample_size
        self._engine: Optional[DenoiseEngine] = None
        self.device = unet.conv_in.weight.device
        self._lora = None                   # imagharmony_b200.lora.LoraWeights once a LoRA is loaded
        self._lora_active: List[Tuple[str, float]] = []
        self._lora_enabled = True
        self._lora_fused: Optional[Dict[str, Dict[str, Tuple[float, float]]]] = None

    # ---- construction ------------------------------------------------------------------------------------------
    @classmethod
    def from_random(cls, cfg: UNetConfig = SDXL_BASE, seed: int = 0, device="cuda", vae_cfg=None):
        """Random-init weights of the given architecture (the benchmark / test configuration)."""
        from imagharmony_b200.vae import AutoencoderKLDecoder
        unet = random_module(UNet2DConditionModel, cfg, seed, device)
        vae = None if vae_cfg is None else random_module(AutoencoderKLDecoder, vae_cfg, seed + 17, device)
        return cls(unet, vae=vae)

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=torch.float16, add_watermarker: bool = False, device="cuda",
                        cfg: Optional[UNetConfig] = None, vae_cfg=None, **kwargs):
        """test.py:68-72.  Loads `<path>/unet/diffusion_pytorch_model.safetensors` (diffusers key names are the native
        UNet's key names, so no key map is needed).  Without `cfg` the UNet's architecture comes from
        `<path>/unet/config.json` when there is one (see _load_pretrained), else it is SDXL-base with the input channel
        count of the checkpoint's conv_in (4, or 9 for the inpainting UNet).  Keywords a subclass needs (the ControlNet
        pipeline's `controlnet`) reach its _from_parts; others are ignored."""
        parts = cls._load_pretrained(path, torch_dtype, device, cfg, vae_cfg)
        return cls._from_parts(parts, device, **kwargs)._configure(parts.index)

    @classmethod
    def _from_parts(cls, parts: _Pretrained, device, **kwargs):
        """The pipeline of this class over the loaded parts."""
        return cls(parts.unet, prompt_encoder=parts.prompt_encoder, vae=parts.vae)

    def _configure(self, index: dict):
        """Per-checkpoint pipeline settings from model_index.json: force_zeros_for_empty_prompt (true for the base,
        false for the refiner: an absent negative prompt is then encoded as "")."""
        if "force_zeros_for_empty_prompt" in index:
            self.force_zeros_for_empty_prompt = bool(index["force_zeros_for_empty_prompt"])
        return self

    @staticmethod
    def _load_pretrained(path: str, torch_dtype, device, cfg: Optional[UNetConfig], vae_cfg) -> _Pretrained:
        """Without `cfg` the UNet's architecture comes from unet/config.json (with model_index.json's
        requires_aesthetics_score: 5 time ids when true) or, without that file, is SDXL-base with the input channel
        count of the checkpoint's conv_in."""
        from safetensors.torch import load_file
        from imagharmony_b200.config import SDXL_VAE
        from imagharmony_b200.vae import AutoencoderKLDecoder
        from .encoders import ClipPromptEncoder
        f = os.path.join(path, "unet", "diffusion_pytorch_model.safetensors")
        if not os.path.exists(f):
            f = os.path.join(path, "unet", "diffusion_pytorch_model.fp16.safetensors")
        if not os.path.exists(f):
            raise FileNotFoundError(f"no SDXL UNet weights under {path}/unet (safetensors)")
        usd = load_file(f)
        index = _read_json(path, "model_index.json")
        meta = _read_json(path, "unet", "config.json")
        if cfg is None and meta:
            cfg = config_from_diffusers(meta, UNetConfig, bool(index.get("requires_aesthetics_score", False)))
        if cfg is None:
            cfg = SDXL_BASE
            if "conv_in.weight" in usd and usd["conv_in.weight"].shape[1] != cfg.in_channels:
                cfg = dataclasses.replace(cfg, in_channels=int(usd["conv_in.weight"].shape[1]))
        unet = UNet2DConditionModel.from_state_dict(cfg, usd, device=device)
        vae = vsd = vcfg = None
        for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
            vf = os.path.join(path, "vae", name)
            if os.path.exists(vf):
                vcfg = vae_cfg or SDXL_VAE
                vmeta = _read_json(path, "vae", "config.json")
                if vae_cfg is None and vmeta:
                    # `force_upcast` decides between the scaled residual stream (the reference's fp32 upcast,
                    # custom_pipelines.py:366-371) and plain fp16 (fp16-fix checkpoints set it to false)
                    vcfg = dataclasses.replace(vcfg, force_upcast=bool(vmeta.get("force_upcast", True)),
                                               scaling_factor=float(vmeta.get("scaling_factor", vcfg.scaling_factor)))
                vsd = load_file(vf)
                vae = AutoencoderKLDecoder.from_state_dict(vcfg, vsd, device=device)  # decoder keys only
                break
        enc = None
        if ClipPromptEncoder.available(path):
            enc = ClipPromptEncoder.from_pretrained(path, device=device, dtype=torch_dtype)
        return _Pretrained(unet, enc, vae, vsd, vcfg, index)

    def to(self, device=None, *args, **kwargs):
        """Weights live on the device the UNet was built on (from_random / from_pretrained take `device=`); moving 5 GB
        of kernel-layout weights behind the caller's back is not offered, a mismatching request raises."""
        if device is not None and not isinstance(device, torch.dtype):
            want = torch.device(device)
            have = torch.device(self.device)
            if want.type != have.type or (want.index is not None and have.index is not None and want.index != have.index):
                raise IHError(f"pipeline was built on {have}; build it with device={want!s} instead of .to({want!s})")
        return self

    def enable_vae_tiling(self):  # test.py:73
        if self.vae is not None:
            self.vae.use_tiling = True

    # ---- reference surface -------------------------------------------------------------------------------------
    def set_scale(self, scale):
        for attn_processor in self.unet.attn_processors.values():           # custom_pipelines.py:17-20
            if isinstance(attn_processor, IPAttnProcessor):
                attn_processor.scale = scale

    # ---- LoRA ([3P] diffusers 0.30 StableDiffusionXLLoraLoaderMixin with the PEFT backend; SURVEY appendix A.8) --
    # Adapters are merged into the canonical fp16 weights of the UNet and the text towers (imagharmony_b200.lora); a
    # pipeline that never loads one runs exactly as without this surface.
    def load_lora_weights(self, pretrained_model_name_or_path_or_dict, weight_name: Optional[str] = None,
                          adapter_name: Optional[str] = None, subfolder: Optional[str] = None, **kwargs):
        """Add a LoRA (a state dict, a .safetensors / .bin file, or a directory -- joined with `subfolder` when given --
        holding `weight_name`) as adapter `adapter_name` (default `default_{i}`); it becomes the only active adapter,
        at weight 1.0.  diffusers' other keywords (hub downloads, caching, loading options) are refused: files are read
        from local paths only."""
        from imagharmony_b200.lora import LoraWeights, prompt_towers, read_state_dict
        if kwargs:
            raise IHError(f"load_lora_weights: keyword arguments {sorted(kwargs)} are not supported (local files, "
                          "weight_name, adapter_name and subfolder only)")
        self._lora_require_unfused("load_lora_weights")
        src = pretrained_model_name_or_path_or_dict
        if subfolder:
            if isinstance(src, dict):
                raise IHError("load_lora_weights: `subfolder` needs a directory, not a state dict")
            src = os.path.join(str(src), subfolder)
        if self._lora is None:
            self._lora = LoraWeights(self.unet, prompt_towers(self.prompt_encoder))
        name = adapter_name or f"default_{len(self._lora.adapters)}"
        if name in self._lora.adapters:
            raise ValueError(f"Adapter name {name} already in use")
        self._lora.add(name, read_state_dict(src, weight_name))
        self._lora_active = [(name, 1.0)]
        self._lora_sync()

    def set_adapters(self, adapter_names, adapter_weights=None):
        """Activate exactly `adapter_names` with `adapter_weights` (a number or one per adapter; default 1.0)."""
        self._lora_require_unfused("set_adapters")
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        self._lora_require_known(names)
        weights = adapter_weights if adapter_weights is not None else 1.0
        weights = list(weights) if isinstance(weights, (list, tuple)) else [weights] * len(names)
        if len(weights) != len(names):
            raise ValueError(f"Length of adapter names {len(names)} is not equal to the length of the weights "
                             f"{len(weights)}")
        self._lora_active = [(n, float(w)) for n, w in zip(names, weights)]
        self._lora_sync()

    def disable_lora(self):
        """Run with the base weights until enable_lora()."""
        self._lora_require_unfused("disable_lora")
        self._lora_enabled = False
        self._lora_sync()

    def enable_lora(self):
        self._lora_require_unfused("enable_lora")
        self._lora_enabled = True
        self._lora_sync()

    def delete_adapters(self, adapter_names):
        self._lora_require_unfused("delete_adapters")
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        self._lora_require_known(names)
        for n in names:
            self._lora.remove(n)
        self._lora_active = [(n, w) for n, w in self._lora_active if n not in names]
        self._lora_sync()
        self._lora.release()

    def unload_lora_weights(self):
        """Remove every adapter (fused ones included): each weight a LoRA touched is its original value again."""
        if self._lora is None:
            return
        for n in list(self._lora.adapters):
            self._lora.remove(n)
        self._lora_active, self._lora_enabled, self._lora_fused = [], True, None
        self._lora_sync()
        self._lora.release()
        self._lora = None

    def get_active_adapters(self) -> List[str]:
        return [n for n, _ in self._lora_active]

    def get_list_adapters(self) -> Dict[str, List[str]]:
        """{"unet": [...], "text_encoder": [...], "text_encoder_2": [...]}: the adapters each component holds."""
        out: Dict[str, List[str]] = {}
        for n in (self._lora.adapters if self._lora is not None else {}):
            for comp in self._lora.components(n):
                out.setdefault(comp, []).append(n)
        return out

    def fuse_lora(self, lora_scale: float = 1.0, fuse_unet: bool = True, fuse_text_encoder: bool = True):
        """Bake the active adapters x `lora_scale` into the weights: until unfuse_lora(), per-call scales have no
        effect and set_adapters raises.  Without a loaded adapter it does nothing; while LoRA is disabled it raises
        (there is no active set to bake: enable_lora() first)."""
        from imagharmony_b200.lora import TE1, TE2, UNET
        self._lora_require_unfused("fuse_lora")
        if self._lora is None or not self._lora.adapters:
            return
        if not self._lora_enabled:
            raise IHError("fuse_lora: LoRA is disabled; call enable_lora() first")
        comps = ([UNET] if fuse_unet else []) + ([TE1, TE2] if fuse_text_encoder else [])
        if comps:
            self._lora_fused = {c: {n: (float(lora_scale), w) for n, w in self._lora_active} for c in comps}
            self._lora_sync()

    def unfuse_lora(self, unfuse_unet: bool = True, unfuse_text_encoder: bool = True):
        """Back to the state before fuse_lora() for the chosen components."""
        from imagharmony_b200.lora import TE1, TE2, UNET
        if self._lora_fused is None:
            return
        for c in ([UNET] if unfuse_unet else []) + ([TE1, TE2] if unfuse_text_encoder else []):
            self._lora_fused.pop(c, None)
        if not self._lora_fused:
            self._lora_fused = None
        self._lora_sync()

    def _lora_require_unfused(self, what: str) -> None:
        if self._lora_fused is not None:
            raise IHError(f"{what}: the LoRA weights are fused; call unfuse_lora() first")

    def _lora_require_known(self, names) -> None:
        have = self._lora.adapters if self._lora is not None else {}
        unknown = [n for n in names if n not in have]
        if unknown:
            raise ValueError(f"Adapter name(s) {unknown} not in the list of present adapters: {list(have)}")

    def _lora_sync(self, components=None, scale: Optional[float] = None) -> None:
        """Merge `components` (default: all) for the active set at the per-call `scale` (None = 1.0); fused components
        keep their baked set."""
        from imagharmony_b200.lora import COMPONENTS
        if self._lora is None:
            return
        s = 1.0 if scale is None else float(scale)
        for comp in components or COMPONENTS:
            if self._lora_fused is not None and comp in self._lora_fused:
                factors = self._lora_fused[comp]
            elif not self._lora_enabled:
                factors = {}
            else:
                factors = {n: (s, w) for n, w in self._lora_active}
            self._lora.sync(comp, factors)

    def _lora_call_scale(self, cross_attention_kwargs: Optional[Dict[str, Any]]) -> Optional[float]:
        """diffusers' `cross_attention_kwargs={"scale": s}`: merges the UNet for s and returns s for encode_prompt's
        lora_scale (None without a loaded LoRA or without a scale)."""
        if self._lora is None:
            return None
        s = cross_attention_kwargs.get("scale") if cross_attention_kwargs else None
        from imagharmony_b200.lora import UNET
        self._lora_sync([UNET], s)
        return s

    @property
    def engine(self) -> DenoiseEngine:
        if self._engine is None or self._engine.scheduler is not self.scheduler:
            # the loop integrates the SAME scheduler object whose init_noise_sigma scaled the initial latents
            self._engine = DenoiseEngine(self.unet, scheduler=self.scheduler)
        return self._engine

    @torch.no_grad()
    def encode_prompt(self, prompt, prompt_2=None, device=None, num_images_per_prompt: int = 1,
                      do_classifier_free_guidance: bool = True, negative_prompt=None, negative_prompt_2=None,
                      prompt_embeds=None, negative_prompt_embeds=None, pooled_prompt_embeds=None,
                      negative_pooled_prompt_embeds=None, lora_scale=None, **kwargs):
        """-> (prompt_embeds [n,77,2048], negative_prompt_embeds, pooled [n,1280], negative_pooled)  ([3P] A.4).
        With a loaded LoRA the text towers run with their deltas scaled by `lora_scale` (None = 1.0); they are merged
        for that scale only when they run (embeddings passed in need no text tower)."""
        if prompt_embeds is None:
            prompts = [prompt] if isinstance(prompt, str) else list(prompt)
            prompt_embeds, pooled_prompt_embeds = self._encode_text(prompts, lora_scale)
            prompt_embeds = prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
            pooled_prompt_embeds = pooled_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
        if do_classifier_free_guidance and negative_prompt_embeds is None and negative_prompt is None \
                and self.force_zeros_for_empty_prompt:
            # [3P] SDXL-base model_index.json: force_zeros_for_empty_prompt = true -> no negative prompt means ZERO embeds
            negative_prompt_embeds = torch.zeros_like(prompt_embeds)
            negative_pooled_prompt_embeds = torch.zeros_like(pooled_prompt_embeds)
        elif do_classifier_free_guidance and negative_prompt_embeds is None:
            negs = negative_prompt if negative_prompt is not None else ""
            negs = [negs] * (prompt_embeds.shape[0] // num_images_per_prompt) if isinstance(negs, str) else list(negs)
            negative_prompt_embeds, negative_pooled_prompt_embeds = self._encode_text(negs, lora_scale)
            negative_prompt_embeds = negative_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
            negative_pooled_prompt_embeds = negative_pooled_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
        return prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds

    def _encode_text(self, prompts, lora_scale):
        if self._lora is not None:
            from imagharmony_b200.lora import TE1, TE2
            self._lora_sync([TE1, TE2], lora_scale)
        return self.prompt_encoder(prompts)

    def prepare_latents(self, batch_size, num_channels_latents, height, width, dtype, device, generator, latents=None):
        """[3P] diffusers prepare_latents: randn * init_noise_sigma; a list of generators draws one sample each."""
        shape = (batch_size, num_channels_latents, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None:
            self._check_batches(batch_size, generator)
            latents = randn_tensor(shape, generator, torch.float32, "cpu")
        latents = latents.to(torch.float32) * self.scheduler.init_noise_sigma
        return latents.to(dtype)

    @torch.no_grad()
    def __call__(self, prompt: Optional[Union[str, List[str]]] = None, prompt_2=None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 50, denoising_end: Optional[float] = None,
                 guidance_scale: float = 5.0, negative_prompt=None, negative_prompt_2=None,
                 num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left=(0, 0), negative_target_size=None,
                 control_guidance_start: float = 0.0, control_guidance_end: float = 1.0, **ignored):
        """Parameter list of custom_pipelines.py:23-56.  Unknown keyword arguments are accepted and ignored, because
        IPAdapterXL.generate forwards a stray `number_class_crossattention=` into this call (test.py:38, demo.py:124)."""
        self._require_latent_unet()
        height, width = self._checked_size(height, width)                             # :189-190
        self._check_callback_steps(callback, callback_steps)
        embeds, sizes = self._embeds_and_sizes(locals(), height, width)               # :192-193, :223, :229-247
        self.scheduler.set_timesteps(num_inference_steps)                             # :250
        lat = self.prepare_latents(embeds[0].shape[0], self.unet.config.in_channels, height, width, torch.float16,
                                   self.device, generator, latents)                  # :255-265
        out = self._denoise_from(lat, num_inference_steps=num_inference_steps, embeds=embeds, sizes=sizes,
                                 guidance_scale=guidance_scale, guidance_rescale=guidance_rescale,
                                 denoising_end=denoising_end, control_guidance_start=control_guidance_start,
                                 control_guidance_end=control_guidance_end, callback=callback,
                                 callback_steps=callback_steps, generator=generator)
        return self._output(out, output_type, return_dict)

    def _checked_size(self, height: Optional[int], width: Optional[int]) -> Tuple[int, int]:
        """The call's height and width (default: the UNet's sample size x 8), refused unless multiples of 8."""
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        if height % 8 or width % 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        return height, width

    def _embeds_and_sizes(self, call: Dict[str, Any], height: int, width: int):
        """-> (encode_prompt's 4 embeddings, `sizes` for _add_time_ids) from the arguments of a pipeline call (its
        locals(): every __call__ takes diffusers' prompt, embedding, LoRA-scale and size parameters under the same
        names).  With a loaded LoRA the UNet is merged for the call's scale first; original_size and target_size
        default to height x width."""
        embeds = self.encode_prompt(call["prompt"], call["prompt_2"], None, call["num_images_per_prompt"],
                                    call["guidance_scale"] > 1.0, call["negative_prompt"], call["negative_prompt_2"],
                                    call["prompt_embeds"], call["negative_prompt_embeds"], call["pooled_prompt_embeds"],
                                    call["negative_pooled_prompt_embeds"],
                                    lora_scale=self._lora_call_scale(call["cross_attention_kwargs"]))
        sizes = (call["original_size"] or (height, width), call["crops_coords_top_left"],
                 call["target_size"] or (height, width), call["negative_original_size"],
                 call["negative_crops_coords_top_left"], call["negative_target_size"])
        return embeds, sizes

    def _denoise_from(self, lat, *, num_inference_steps: int, embeds, sizes, guidance_scale, guidance_rescale,
                      generator, callback, callback_steps, t_start: int = 0, denoising_end=None,
                      control_guidance_start=0.0, control_guidance_end=1.0, inpaint=None, unet_cond=None,
                      controlnet=None, aesthetic=None, adapter=None) -> torch.Tensor:
        """The loop over timesteps[t_start:], truncated by denoising_end (:307-316), from the noised start latents `lat`
        with the IP scale of the processors (:319-322); the micro-conditioning time ids are formed from `sizes`, and
        from `aesthetic` = (aesthetic_score, negative_aesthetic_score) for a 5-id UNet. -> final latents."""
        add_time_ids, negative_add_time_ids = self._add_time_ids(embeds[0].shape[0], sizes, aesthetic)
        loop_end = self._loop_end(num_inference_steps, denoising_end, t_start)
        conditioning_scale = self._ip_scale()
        if loop_end > t_start:
            out = self.engine.run(lat, *embeds, add_time_ids, num_inference_steps,
                                  guidance_scale=guidance_scale, ip_scale=conditioning_scale,
                                  control_guidance_start=control_guidance_start,
                                  control_guidance_end=control_guidance_end, guidance_rescale=guidance_rescale,
                                  num_loop_steps=loop_end, callback=callback, callback_steps=callback_steps,
                                  negative_time_ids=negative_add_time_ids, begin_step=t_start, inpaint=inpaint,
                                  generator=generator, unet_cond=unet_cond, controlnet=controlnet, adapter=adapter)
        else:
            out = lat.to(self.device)
        self.set_scale(conditioning_scale)
        return out

    def _loop_end(self, num_inference_steps: int, denoising_end, t_start: int = 0) -> int:
        """The schedule index the loop over timesteps[t_start:] stops at: num_inference_steps, or with a valid
        denoising_end (:307-316) t_start + the number of those timesteps at or above its cutoff.  The scheduler's
        timesteps must be set."""
        if not _fraction(denoising_end):
            return num_inference_steps
        cutoff = _denoising_cutoff(self.scheduler.num_train_timesteps, denoising_end)
        return t_start + int(sum(1 for t in self.scheduler.timesteps[t_start:] if t >= cutoff))

    @staticmethod
    def _check_batches(batch_size: int, generator, *batches: Tuple[str, int]) -> None:
        """Refuses, before anything is encoded or drawn, an input batch ((description, size) in `batches`) that does
        not divide the prompt batch, then a list of generators that is not one per prompt-batch entry."""
        for what, n in batches:
            if batch_size % n:
                raise ValueError(f"cannot duplicate {what} batch of {n} to a prompt batch of {batch_size}")
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"got {len(generator)} generators for a batch of {batch_size}")

    @staticmethod
    def _check_callback_steps(callback, callback_steps) -> None:
        if callback is not None and (not isinstance(callback_steps, int) or callback_steps <= 0):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps}")   # [3P] check_inputs

    def _refuse_unsupported(self, given: Dict[str, Any]) -> None:
        """Raises IHError for the arguments in UNSUPPORTED that `given` sets."""
        refused = [k for k in self.UNSUPPORTED if given.get(k) is not None]
        if refused:
            raise IHError(f"{type(self).__name__} does not implement {refused}")

    @staticmethod
    def _add_time_ids(batch: int, sizes, aesthetic=None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """:277-294 [3P] _get_add_time_ids: (positive, negative or None) micro-conditioning ids [batch, 6] from `sizes` =
        (original_size, crops_coords_top_left, target_size, negative_original_size, negative_crops_coords_top_left,
        negative_target_size); requires_aesthetics_score = False.  With `aesthetic` = (aesthetic_score,
        negative_aesthetic_score) it is the image-to-image requires_aesthetics_score = True form, [batch, 5] each:
        original_size + crops + (aesthetic_score,) and negative_original_size (default: original_size) +
        negative_crops + (negative_aesthetic_score,)."""
        original_size, crops, target_size, neg_original_size, neg_crops, neg_target_size = sizes

        def time_ids(size, crop, target):
            return torch.tensor([list(size) + list(crop) + list(target)], dtype=torch.float32).repeat(batch, 1)
        if aesthetic is not None:
            score, neg_score = aesthetic
            return (time_ids(original_size, crops, [score]),
                    time_ids(neg_original_size or original_size, neg_crops, [neg_score]))
        negative = None
        if neg_original_size is not None and neg_target_size is not None:
            negative = time_ids(neg_original_size, neg_crops, neg_target_size)
        return time_ids(original_size, crops, target_size), negative

    def _ip_scale(self) -> float:
        """The IP scale of the first image-prompt processor (:319-322), 1.0 without one."""
        for attn_processor in self.unet.attn_processors.values():
            if isinstance(attn_processor, IPAttnProcessor):
                return attn_processor.scale
        return 1.0

    def _require_latent_unet(self) -> None:
        """Text-to-image and image-to-image have no mask to feed the 9-channel inpainting UNet."""
        if self.unet.config.in_channels != 4:
            raise IHError(f"{type(self).__name__} needs a 4-channel UNet (this one has {self.unet.config.in_channels} "
                          "input channels); the 9-channel inpainting UNet runs in StableDiffusionXLInpaintPipeline")

    def _output(self, out: torch.Tensor, output_type: Optional[str], return_dict: bool):
        """Final latents -> images (:365-386) in the requested output type."""
        if output_type == "latent":
            image = out
        else:
            if self.vae_decode is not None:
                image = self.vae_decode(out / 0.13025, output_type)                   # :373 (scaling_factor [3P])
            elif self.vae is not None:
                from imagharmony_b200.vae import postprocess
                image = postprocess(self.vae.decode(out), output_type)                # :373 + :383 (/ scaling_factor folded)
            else:
                raise IHError("this pipeline has no VAE decoder: call with output_type='latent', build it with a `vae` "
                              "(from_random(vae_cfg=...), from_pretrained with a vae/ folder) or pass a vae_decode callable")
        if not return_dict:
            return (image,)
        return StableDiffusionXLPipelineOutput(images=image)


def preprocess_image(image, vae_scale_factor: int = 8, height: Optional[int] = None,
                     width: Optional[int] = None) -> torch.Tensor:
    """[3P] diffusers VaeImageProcessor.preprocess (SDXL defaults: resize with Lanczos, normalise): PIL image(s) ->
    float32 [B, 3, H, W] in [-1, 1] with H, W floored to multiples of `vae_scale_factor` (every image takes the first
    one's size), or the requested `height` x `width` when both are given.  A [B, 3, H, W] / [3, H, W] tensor is taken
    as it is, resized (nearest) when its size is not a multiple of the factor or not the requested one; as in diffusers
    it is expected in [-1, 1], and one without negative values is taken as [0, 1] and normalised."""
    def size(h, w):
        if height is not None and width is not None:
            return height, width
        return h - h % vae_scale_factor, w - w % vae_scale_factor
    x = _load_images(image, size, "image", vae_scale_factor)
    return x * 2.0 - 1.0 if x.min() >= 0 else x           # PIL images are in [0, 1]: always normalised


class StableDiffusionXLImg2ImgPipeline(StableDiffusionXLCustomPipeline):
    """Image-to-image with the call surface of [3P] diffusers `StableDiffusionXLImg2ImgPipeline`, so that
    `IPAdapterXL(img2img_pipe, ...).generate(pil_image=..., image=init, strength=s)` works as it does on the
    reference built over that pipeline.  The init image is encoded by the native VAE encoder
    (imagharmony_b200.vae.AutoencoderKLEncoder), its posterior sampled and noised to sigma[t_start] by one kernel
    (ops.vae_posterior_noise), and the denoise loop runs over timesteps[t_start:] on the same engine and graphs as
    text-to-image (DenoiseEngine.run(begin_step=t_start)).

    Batch expansion follows diffusers: with one generator the encoded latents of the image batch are tiled to the
    prompt batch with torch.cat (prompt slot b gets image b % n_images, while num_images_per_prompt repeats prompts
    in place), with a list of generators each slot encodes image b % n_images with its own generator.
    The SDXL-base configuration has requires_aesthetics_score = False: `aesthetic_score` / `negative_aesthetic_score`
    are accepted and unused.  A UNet with 5 micro-conditioning ids (the SDXL refiner, unet.config.num_time_ids = 5)
    requires them: its time ids are original_size + crops + (aesthetic_score,) for the positive half and
    negative_original_size + negative_crops + (negative_aesthetic_score,) for the negative one.

    Ensemble of experts ([3P] diffusers `denoising_start`): the base runs with `denoising_end=d, output_type="latent"`,
    and this pipeline (usually on the refiner) finishes with `image=<those latents>, denoising_start=d`.  A [B, 4, h, w]
    `image` is taken as latents: not encoded, scaled or noised, no random draw, tiled to the prompt batch like encoded
    latents; the loop runs the last n timesteps, those below the cutoff int(round(1000 - d * 1000)), on the same engine
    and graphs (DenoiseEngine.run(begin_step=T - n)), and returns the latents unchanged when n = 0.  `strength` is
    validated and unused.  Latents need a valid `denoising_start` (a float in (0, 1); other values are ignored, as in
    diffusers), and `denoising_start` needs latents: a pixel image with it (encoded without noise) is not implemented;
    both raise IHError."""

    # diffusers arguments that change the result and have no native implementation: refused, never ignored
    UNSUPPORTED = ("timesteps", "sigmas", "latents", "ip_adapter_image", "ip_adapter_image_embeds",
                   "clip_skip", "callback_on_step_end")
    TIME_IDS = (5, 6)

    def __init__(self, unet: UNet2DConditionModel, prompt_encoder: Optional[Callable] = None,
                 vae_decode: Optional[Callable] = None,
                 scheduler: Optional[Union[EulerDiscreteScheduler, DPMSolverMultistepScheduler,
                                            UniPCMultistepScheduler]] = None, vae=None,
                 vae_encoder=None):
        super().__init__(unet, prompt_encoder=prompt_encoder, vae_decode=vae_decode, scheduler=scheduler, vae=vae)
        self.vae_encoder = vae_encoder      # imagharmony_b200.vae.AutoencoderKLEncoder or None

    @classmethod
    def from_random(cls, cfg: UNetConfig = SDXL_BASE, seed: int = 0, device="cuda", vae_cfg=None):
        """Random-init weights; with `vae_cfg` also a random VAE decoder and encoder."""
        pipe = super().from_random(cfg, seed=seed, device=device, vae_cfg=vae_cfg)
        if vae_cfg is not None:
            from imagharmony_b200.vae import AutoencoderKLEncoder
            pipe.vae_encoder = random_module(AutoencoderKLEncoder, vae_cfg, seed + 19, device)
        return pipe

    @classmethod
    def _from_parts(cls, parts: _Pretrained, device, **kwargs):
        """The VAE checkpoint also provides the encoder."""
        pipe = super()._from_parts(parts, device)
        if parts.vae_state is not None:
            from imagharmony_b200.vae import AutoencoderKLEncoder
            pipe.vae_encoder = AutoencoderKLEncoder.from_state_dict(parts.vae_config, parts.vae_state, device=device)
        return pipe

    def enable_vae_tiling(self):
        super().enable_vae_tiling()
        if self.vae_encoder is not None:
            self.vae_encoder.use_tiling = True

    def prepare_img2img_latents(self, image: torch.Tensor, batch_size: int, generator, sigma: float) -> torch.Tensor:
        """[3P] StableDiffusionXLImg2ImgPipeline.prepare_latents (fp16 latents): encode, sample the posterior, scale,
        add_noise(sigma).  eps (fp32 when the VAE config asks for the upcast, else fp16) and the fp16 noise are drawn
        here from the caller's generator(s) in diffusers' order; the arithmetic is one kernel."""
        n_img = image.shape[0]
        self._check_batches(batch_size, generator, ("an image", n_img))
        # with a list, every generator samples the posterior of the image of its batch slot
        sample, noise = self._encode_posterior(image, batch_size if isinstance(generator, list) else n_img, generator,
                                               batch_size)
        return sample(noise, sigma)

    def prepare_handoff_latents(self, latents: torch.Tensor, batch_size: int) -> torch.Tensor:
        """[3P] StableDiffusionXLImg2ImgPipeline.prepare_latents(add_noise=False) for a latent `image`: the latents as
        they are (fp16 on the device), tiled to the prompt batch with torch.cat like encoded latents."""
        n_img = latents.shape[0]
        self._check_batches(batch_size, None, ("a latent", n_img))
        lat = latents.to(self.device, torch.float16)
        return lat.repeat(batch_size // n_img, 1, 1, 1) if batch_size > n_img else lat

    def _encode_posterior(self, image: torch.Tensor, n_eps: int, generator, noise_batch: Optional[int] = None):
        """Encodes `image` and draws the posterior eps of n_eps images (_posterior_eps), then, given noise_batch, the
        fp16 noise [noise_batch, 4, h, w]: both from `generator` in diffusers' order.  -> (sample, noise or None), where
        sample(x, sigma) is the scaled posterior sample + x * sigma for a [B, 4, h, w] x, fp16 on the device, in one
        kernel (ops.vae_posterior_noise; slot b samples image b % n_eps).  Zero x and sigma 0 give the clean latents
        exactly (fp16(zs + 0) = zs)."""
        venc = self.vae_encoder
        moments = venc.encode_moments_nhwc(image.to(self.device, torch.float16))      # [n_img, h, w, 16]
        L, sf, h, w = venc.config.latent_channels, venc.config.scaling_factor, moments.shape[1], moments.shape[2]
        eps = self._posterior_eps(n_eps, h, w, generator)
        noise = None
        if noise_batch is not None:
            noise = randn_tensor((noise_batch, L, h, w), generator, torch.float16, self.device, "cpu")
        return (lambda x, sigma: ops.vae_posterior_noise(moments, eps, x, L, sf, sigma)), noise

    def _posterior_eps(self, n: int, h: int, w: int, generator) -> torch.Tensor:
        """The posterior draw of [3P] diffusers' `_encode_vae_image(images, generator)` for n images with latents of
        h x w: image i with generator[i] for a list, fp32 when the VAE is upcast (else fp16), on the generator's device
        (the CPU without one); -> on the device.  For the masked images (image * (mask < 0.5) broadcast over both
        batches) 4-channel inpainting draws and drops it (SURVEY C.31); the 9-channel path encodes with it, and with the
        same draw of the image batch (SURVEY C.32)."""
        cfg = self.vae_encoder.config
        dtype = torch.float32 if getattr(cfg, "force_upcast", True) else torch.float16
        return randn_tensor((n, cfg.latent_channels, h, w), generator, dtype, self.device, "cpu")

    @torch.no_grad()
    def __call__(self, prompt: Optional[Union[str, List[str]]] = None, prompt_2=None, image=None, strength: float = 0.3,
                 num_inference_steps: int = 50, denoising_end: Optional[float] = None, guidance_scale: float = 5.0,
                 negative_prompt=None, negative_prompt_2=None, num_images_per_prompt: Optional[int] = 1,
                 eta: float = 0.0, generator=None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left=(0, 0), negative_target_size=None, aesthetic_score: float = 6.0,
                 negative_aesthetic_score: float = 2.5, control_guidance_start: float = 0.0,
                 control_guidance_end: float = 1.0, denoising_start: Optional[float] = None, **kwargs):
        """The text-to-image parameter list without height / width, plus `image` (PIL image(s) or a [B, 3, H, W]
        tensor in [-1, 1], or [B, 4, h, w] latents with `denoising_start`), `strength` and `denoising_start`.  Unknown
        keywords are ignored as in the text-to-image pipeline, except the diffusers arguments in UNSUPPORTED, which
        raise IHError."""
        self._require_euler()
        self._require_latent_unet()
        self._refuse_unsupported(kwargs)
        start = denoising_start if _fraction(denoising_start) else None
        if start is not None and _fraction(denoising_end) and start >= denoising_end:
            raise ValueError(f"`denoising_start`: {start} cannot be larger than or equal to `denoising_end`: "
                             f"{denoising_end} when using type float.")
        handoff = isinstance(image, torch.Tensor) and image.dim() == 4 and image.shape[1] == self.unet.config.out_channels
        if handoff != (start is not None):
            raise IHError("a latent `image` [B, 4, h, w] needs `denoising_start` as a float in (0, 1)" if handoff else
                          "`denoising_start` continues from latents (`image` [B, 4, h, w], e.g. a base run's "
                          "output_type='latent' with denoising_end); a pixel image with denoising_start is not implemented")
        if start is None:
            t_start = self._begin_index(num_inference_steps, strength)
        elif not 0.0 <= strength <= 1.0:
            raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
        self._check_callback_steps(callback, callback_steps)
        if image is None:
            raise ValueError("`image` input cannot be undefined")
        if handoff:
            height, width = image.shape[2] * self.vae_scale_factor, image.shape[3] * self.vae_scale_factor
        else:
            self._require_vae_encoder()
            pixels = preprocess_image(image, self.vae_scale_factor)
            height, width = pixels.shape[2], pixels.shape[3]
        require_latent_size(self.unet.config, height // self.vae_scale_factor, width // self.vae_scale_factor)
        embeds, sizes = self._embeds_and_sizes(locals(), height, width)
        self.scheduler.set_timesteps(num_inference_steps)
        if handoff:
            t_start = denoising_start_begin_step(self.scheduler.timesteps, self.scheduler.num_train_timesteps, start)
            lat = self.prepare_handoff_latents(image, embeds[0].shape[0])
        else:
            lat = self.prepare_img2img_latents(pixels, embeds[0].shape[0], generator,
                                               self.scheduler.add_noise_sigma(t_start))
        aesthetic = (aesthetic_score, negative_aesthetic_score) if self.unet.config.num_time_ids == 5 else None
        out = self._denoise_from(lat, t_start=t_start, num_inference_steps=num_inference_steps, embeds=embeds,
                                 sizes=sizes, guidance_scale=guidance_scale, guidance_rescale=guidance_rescale,
                                 denoising_end=denoising_end, control_guidance_start=control_guidance_start,
                                 control_guidance_end=control_guidance_end, callback=callback,
                                 callback_steps=callback_steps, generator=generator, aesthetic=aesthetic)
        return self._output(out, output_type, return_dict)

    def _require_vae_encoder(self) -> None:
        """Encoding a pixel image needs the KL VAE encoder.  With a tiny autoencoder as `pipe.vae` diffusers encodes
        with the tiny encoder, which is not built here; encoding with the KL encoder instead would silently give other
        latents.  Latent hand-overs (`denoising_start`) encode nothing and run."""
        from imagharmony_b200.taesd import AutoencoderTinyDecoder
        if isinstance(self.vae, AutoencoderTinyDecoder):
            raise IHError(f"{type(self).__name__}: encoding a pixel image with a tiny autoencoder (AutoencoderTiny) as "
                          "pipe.vae is not implemented; keep the KL VAE for this call, or pass latents with "
                          "denoising_start")
        if self.vae_encoder is None:
            raise IHError("this pipeline has no VAE encoder: build it with from_random(vae_cfg=...) or from_pretrained "
                          "with a vae/ folder")

    def _require_euler(self) -> None:
        """Image-to-image and inpainting noise the image latents with Euler's add_noise (x + sigma * noise) inside the
        posterior kernel; DPM-Solver++ and UniPC noise in VP form (alpha * x + sigma_vp * noise), which it does not
        compute."""
        if isinstance(self.scheduler, (DPMSolverMultistepScheduler, UniPCMultistepScheduler)):
            raise IHError(f"{type(self).__name__} supports EulerDiscreteScheduler and EulerAncestralDiscreteScheduler; "
                          f"{type(self.scheduler).__name__} runs text-to-image (StableDiffusionXLCustomPipeline)")

    def _begin_index(self, num_inference_steps: int, strength: float) -> int:
        """[3P] check_inputs and get_timesteps: the schedule index t_start a run of `strength` begins at."""
        if not 0.0 <= strength <= 1.0:
            raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
        t_start = self.scheduler.img2img_begin_index(num_inference_steps, strength)
        if num_inference_steps - t_start < 1:
            raise ValueError(f"After adjusting the num_inference_steps by strength parameter: {strength}, the number of "
                             f"pipeline steps is {num_inference_steps - t_start} which is < 1 and not appropriate for "
                             "this pipeline.")
        return t_start


def preprocess_mask(mask, height: int, width: int) -> torch.Tensor:
    """[3P] diffusers VaeImageProcessor(do_normalize=False, do_binarize=True, do_convert_grayscale=True).preprocess:
    PIL mask(s) are converted to "L", resized to width x height with Lanczos and divided by 255; a [B, 1, H, W],
    [B, H, W] or [H, W] tensor in [0, 1] is resized with nearest interpolation.  Then binarized (< 0.5 -> 0, else 1).
    -> float32 [B, 1, height, width]."""
    import numpy as np
    from PIL import Image
    masks = _pil_list(mask)
    if masks is not None:
        masks = [m.convert("L").resize((width, height), resample=Image.LANCZOS) for m in masks]
        x = torch.from_numpy(np.stack([np.array(m).astype(np.float32) / 255.0 for m in masks]))[:, None]
    elif isinstance(mask, torch.Tensor):
        x = mask.float()
        if x.dim() == 2:
            x = x[None, None]
        elif x.dim() == 3:
            x = x[:, None]
        if x.dim() != 4 or x.shape[1] != 1:
            raise ValueError(f"mask tensor must be [B, 1, H, W], [B, H, W] or [H, W], got {tuple(mask.shape)}")
        x = torch.nn.functional.interpolate(x, size=(height, width))
    else:
        raise ValueError(f"`mask_image` must be a PIL image, a list of them or a tensor, got {type(mask).__name__}")
    return (x >= 0.5).float().contiguous()


class StableDiffusionXLInpaintPipeline(StableDiffusionXLImg2ImgPipeline):
    """Inpainting with the call surface of [3P] diffusers `StableDiffusionXLInpaintPipeline` over the 4-channel SDXL-base
    UNet, so that `IPAdapterXL(inpaint_pipe, ...).generate(pil_image=..., image=init, mask_image=mask, strength=s)`
    works as it does on the reference built over that pipeline.  The region where the mask is 1 is regenerated; after
    every step the rest is replaced by the image latents re-noised to the next sigma (the clean latents after the last
    step), fused into the step kernel (ops.euler_inpaint_step, DenoiseEngine.run(inpaint=...)).

    Differences from image-to-image follow diffusers: defaults strength = 0.9999 (the first step is skipped) and
    guidance_scale = 7.5; height / width default to the UNet's sample size x 8, not to the image's size, and the image
    and the mask are resized to them.  Image and mask batches are tiled to the prompt batch with `repeat` (slot b gets
    image b % n_images and mask b % n_masks); with a list of generators only the first n_images encode (SURVEY C.19).

    With the 9-channel inpainting UNet (diffusers' stable-diffusion-xl-1.0-inpainting-0.1; `from_pretrained` reads the
    channel count from the checkpoint) there is no blend: every step the UNet sees the latents, the mask and the latents
    of the masked image (image * (mask < 0.5)), which conv_in reads from a static buffer next to the step's latents
    (DenoiseEngine.run(unet_cond=...)).  At strength 1 the image itself is not encoded (SURVEY C.32).
    `padding_mask_crop` is not implemented and raises IHError, as does a UNet with any other channel count."""

    UNSUPPORTED = StableDiffusionXLImg2ImgPipeline.UNSUPPORTED + ("denoising_start", "masked_image_latents",
                                                                  "padding_mask_crop")
    TIME_IDS = (6,)

    def prepare_inpaint_latents(self, image: torch.Tensor, batch_size: int, generator, t_start: int,
                                is_strength_max: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """[3P] StableDiffusionXLInpaintPipeline.prepare_latents (return_image_latents, fp16 latents) ->
        (start latents, clean image latents, noise), each [batch_size, 4, h, w] fp16 on the device.  The posterior
        kernel gives the clean latents (_encode_posterior) and, with the noise and sigma[t_start], the start latents
        (add_noise); at strength 1 the start is noise * init_noise_sigma."""
        n_img = image.shape[0]
        self._check_batches(batch_size, generator, ("an image", n_img))
        # _encode_vae_image samples the n_img images with generator[i] before the batch is tiled
        sample, noise = self._encode_posterior(image, n_img, generator, batch_size)
        image_latents = sample(torch.zeros_like(noise), 0.0)
        if is_strength_max:
            latents = (noise.float() * self.scheduler.init_noise_sigma).half()
        else:
            latents = sample(noise, self.scheduler.add_noise_sigma(t_start))
        return latents, image_latents, noise

    @torch.no_grad()
    def __call__(self, prompt: Optional[Union[str, List[str]]] = None, prompt_2=None, image=None, mask_image=None,
                 height: Optional[int] = None, width: Optional[int] = None, padding_mask_crop: Optional[int] = None,
                 strength: float = 0.9999, num_inference_steps: int = 50, denoising_end: Optional[float] = None,
                 guidance_scale: float = 7.5, negative_prompt=None, negative_prompt_2=None,
                 num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left=(0, 0), negative_target_size=None, aesthetic_score: float = 6.0,
                 negative_aesthetic_score: float = 2.5, control_guidance_start: float = 0.0,
                 control_guidance_end: float = 1.0, **kwargs):
        """The image-to-image parameter list plus `mask_image` (PIL image(s) or a tensor in [0, 1]; 1 = regenerate),
        `height`, `width` and `padding_mask_crop`.  Unknown keywords are ignored, except the diffusers arguments in
        UNSUPPORTED and a `padding_mask_crop`, which raise IHError."""
        self._require_euler()
        self._refuse_unsupported({**kwargs, "padding_mask_crop": padding_mask_crop})
        unet9 = self.unet.config.in_channels == 9 and self.unet.conv_in.weight.shape[1] == 9
        if self.unet.config.in_channels != 4 and not unet9:
            raise IHError(f"StableDiffusionXLInpaintPipeline supports the 4-channel UNet and the 9-channel inpainting "
                          f"UNet (this one has config.in_channels = {self.unet.config.in_channels} and a conv_in of "
                          f"{self.unet.conv_in.weight.shape[1]} input channels)")
        t_start = self._begin_index(num_inference_steps, strength)
        height, width = self._checked_size(height, width)
        self._check_callback_steps(callback, callback_steps)
        if image is None or mask_image is None:
            raise ValueError("`image` and `mask_image` inputs cannot be undefined")
        self._require_vae_encoder()
        pixels = preprocess_image(image, self.vae_scale_factor, height, width)
        mask = preprocess_mask(mask_image, height, width)
        embeds, sizes = self._embeds_and_sizes(locals(), height, width)
        batch = embeds[0].shape[0]
        self.scheduler.set_timesteps(num_inference_steps)
        if unet9:
            lat, mask_lat, masked_lat = self.prepare_inpaint9_inputs(pixels, mask, batch, generator, t_start,
                                                                     strength == 1.0)
            cond = dict(unet_cond=(mask_lat, masked_lat))
        else:
            # the mask's batch is refused before the encode, after the image's and the generators' checks
            self._check_batches(batch, generator, ("an image", pixels.shape[0]))
            self._check_batches(batch, None, ("a mask", mask.shape[0]))
            lat, image_latents, noise = self.prepare_inpaint_latents(pixels, batch, generator, t_start, strength == 1.0)
            # the masked image's latents only feed a 9-channel UNet: with 4 channels diffusers encodes them unused.
            # That encode is skipped; its posterior draw comes after the noise, so it changes only what is drawn later:
            # the step noise of Euler Ancestral, for which the draw is made and dropped (SURVEY C.31)
            h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
            if isinstance(self.scheduler, EulerAncestralDiscreteScheduler):
                self._posterior_eps(max(pixels.shape[0], mask.shape[0]), h, w, generator)
            mask_lat = torch.nn.functional.interpolate(mask, size=(h, w)).half()
            mask_lat = mask_lat.repeat(batch // mask_lat.shape[0], 1, 1, 1).to(self.device)
            cond = dict(inpaint=(image_latents, noise, mask_lat))
        out = self._denoise_from(lat, t_start=t_start, num_inference_steps=num_inference_steps, embeds=embeds,
                                 sizes=sizes, guidance_scale=guidance_scale, guidance_rescale=guidance_rescale,
                                 denoising_end=denoising_end, control_guidance_start=control_guidance_start,
                                 control_guidance_end=control_guidance_end, callback=callback,
                                 callback_steps=callback_steps, generator=generator, **cond)
        return self._output(out, output_type, return_dict)

    def prepare_inpaint9_inputs(self, image: torch.Tensor, mask: torch.Tensor, batch_size: int, generator, t_start: int,
                                is_strength_max: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """[3P] StableDiffusionXLInpaintPipeline.prepare_latents (return_image_latents=False) and prepare_mask_latents
        for the 9-channel UNet -> (start latents [batch_size, 4, h, w], mask [batch_size, 1, h, w], masked-image latents
        [batch_size, 4, h, w]), fp16 on the device, CFG halves not yet formed.  Per generator the draws come in
        diffusers' order: the image's posterior eps (strength < 1 only: at strength 1 the image is not encoded), the
        noise, then the masked images' posterior eps (SURVEY C.32).  Both encodes use the posterior kernel
        (_encode_posterior)."""
        n_img, n_mask = image.shape[0], mask.shape[0]
        if n_img != n_mask and 1 not in (n_img, n_mask):
            raise ValueError(f"an image batch of {n_img} and a mask batch of {n_mask} do not broadcast")
        n_masked = max(n_img, n_mask)
        self._check_batches(batch_size, generator, ("a image", n_img), ("a mask", n_mask), ("a masked image", n_masked))
        shape = (batch_size, self.vae_encoder.config.latent_channels, image.shape[2] // self.vae_scale_factor,
                 image.shape[3] // self.vae_scale_factor)
        if is_strength_max:
            noise = randn_tensor(shape, generator, torch.float16, self.device, "cpu")
            latents = (noise.float() * self.scheduler.init_noise_sigma).half()
        else:
            sample, noise = self._encode_posterior(image, n_img, generator, batch_size)
            latents = sample(noise, self.scheduler.add_noise_sigma(t_start))
        sample, _ = self._encode_posterior(image * (mask < 0.5), n_masked, generator)
        masked_latents = sample(torch.zeros_like(noise), 0.0)
        mask_lat = torch.nn.functional.interpolate(mask, size=shape[2:]).half()
        return latents, mask_lat.repeat(batch_size // n_mask, 1, 1, 1).to(self.device), masked_latents


def preprocess_control_image(image, height: Optional[int] = None, width: Optional[int] = None,
                             vae_scale_factor: int = 8) -> torch.Tensor:
    """[3P] diffusers VaeImageProcessor(do_convert_rgb=True, do_normalize=False).preprocess, the ControlNet pipeline's
    control-image processor: PIL image(s) -> RGB, Lanczos resize to width x height, / 255; a [B, 3, H, W] / [3, H, W]
    tensor in [0, 1] is resized with nearest interpolation.  Without height / width the first image's size floored to
    multiples of `vae_scale_factor` is used.  -> float32 [B, 3, height, width] in [0, 1]."""
    def size(h, w):
        return (height if height is not None else h - h % vae_scale_factor,
                width if width is not None else w - w % vae_scale_factor)
    return _load_images(image, size, "control image", vae_scale_factor)


class StableDiffusionXLControlNetPipeline(StableDiffusionXLCustomPipeline):
    """Text-to-image with one SDXL ControlNet, with the call surface of [3P] diffusers
    `StableDiffusionXLControlNetPipeline`, so that `IPAdapterXL(controlnet_pipe, ...).generate(pil_image=...,
    image=control, controlnet_conditioning_scale=s)` works as on the reference (ip_adapter.py:128-133 installs
    CNAttnProcessor on `pipe.controlnet`).  Every step runs the ControlNet and adds its residuals to the UNet's skip
    connections inside the replayed step graph (DenoiseEngine.run(controlnet=...)).

    Note: here `control_guidance_start` / `control_guidance_end` gate the CONTROLNET (it runs at step i only when
    i/T >= start and (i+1)/T <= end), as in diffusers' ControlNet pipeline -- not the IP-adapter scale, which the
    reference's text-to-image pipeline gates with the same names (custom_pipelines.py:326-329).  The IP scale is not
    gated here.

    `controlnet` may also be a list of ControlNetModels, wrapped in a MultiControlNetModel as diffusers does, or a
    MultiControlNetModel.  Then `image` is a list with one control image per net, `controlnet_conditioning_scale` a
    float (broadcast to every net) or a list, and `control_guidance_start` / `end` floats or lists, aligned as in
    diffusers 0.30; each net runs only inside its own window, and the active nets' residuals are summed.

    `global_pool_conditions` models, ControlNet image-to-image / inpainting, several conditionings per batch entry,
    `denoising_end` and the diffusers arguments in UNSUPPORTED raise IHError (ValueError for nested image lists)."""

    UNSUPPORTED = ("denoising_end", "timesteps", "sigmas", "ip_adapter_image", "ip_adapter_image_embeds", "clip_skip",
                   "callback_on_step_end", "strength", "mask_image")

    def __init__(self, unet: UNet2DConditionModel, controlnet, prompt_encoder: Optional[Callable] = None,
                 vae_decode: Optional[Callable] = None, scheduler=None, vae=None):
        from imagharmony_b200.controlnet import MultiControlNetModel
        if isinstance(controlnet, (list, tuple)):          # [3P] diffusers wraps a list the same way
            controlnet = MultiControlNetModel(controlnet)
        super().__init__(unet, prompt_encoder=prompt_encoder, vae_decode=vae_decode, scheduler=scheduler, vae=vae)
        self.controlnet = controlnet

    @classmethod
    def from_random(cls, cfg: UNetConfig = SDXL_BASE, controlnet_cfg: ControlNetConfig = SDXL_CONTROLNET, seed: int = 0,
                    device="cuda", vae_cfg=None):
        """Random-init UNet and ControlNet weights (every weight random, zero convs included).  A list of ControlNet
        configs gives a Multi-ControlNet pipeline, net j seeded with seed + 23 + 7j."""
        from imagharmony_b200.controlnet import ControlNetModel
        base = StableDiffusionXLCustomPipeline.from_random(cfg, seed=seed, device=device, vae_cfg=vae_cfg)
        cfgs = controlnet_cfg if isinstance(controlnet_cfg, (list, tuple)) else [controlnet_cfg]
        nets = [random_module(ControlNetModel, c, seed + 23 + 7 * j, device) for j, c in enumerate(cfgs)]
        return cls(base.unet, nets if isinstance(controlnet_cfg, (list, tuple)) else nets[0], vae=base.vae)

    @classmethod
    def from_pretrained(cls, path: str, controlnet=None, torch_dtype=torch.float16, add_watermarker: bool = False,
                        device="cuda", cfg: Optional[UNetConfig] = None, vae_cfg=None, **kwargs):
        """`controlnet=ControlNetModel.from_pretrained(dir)` (or a list of them, or a MultiControlNetModel) with the
        SDXL folder `path` of StableDiffusionXLCustomPipeline.from_pretrained; refused before anything is read
        without it."""
        if controlnet is None:
            raise ValueError("StableDiffusionXLControlNetPipeline.from_pretrained needs controlnet=")
        return super().from_pretrained(path, torch_dtype, add_watermarker, device, cfg, vae_cfg, controlnet=controlnet)

    @classmethod
    def _from_parts(cls, parts: _Pretrained, device, controlnet=None, **kwargs):
        return cls(parts.unet, controlnet, prompt_encoder=parts.prompt_encoder, vae=parts.vae)

    def _align_multi(self, image, scale, start, end):
        """[3P] diffusers 0.30 for a MultiControlNetModel: scalar guidance start / end become lists (the length of the
        other list, or one entry per net), a float scale is broadcast; `image` must be a flat list with one entry per
        net.  -> (images, scales, starts, ends), one entry per net."""
        k = len(self.controlnet.nets)
        if not isinstance(image, list):
            raise TypeError("For multiple controlnets: `image` must be type `list`")
        if any(isinstance(i, list) for i in image):
            raise ValueError("A single batch of multiple conditionings is not supported: pass one image (or one "
                             "batch tensor / list of PIL images) per ControlNet, not a nested list")
        if len(image) != k:
            raise ValueError(f"For multiple controlnets: `image` must have one entry per ControlNet, got {len(image)} "
                             f"images and {k} ControlNets")
        if isinstance(scale, (list, tuple)):
            if any(isinstance(s, (list, tuple)) for s in scale):
                raise ValueError("A single batch of multiple conditionings is not supported: "
                                 "`controlnet_conditioning_scale` must be a flat list")
            if len(scale) != k:
                raise ValueError(f"`controlnet_conditioning_scale` has {len(scale)} entries for {k} ControlNets")
            scales = [float(s) for s in scale]
        else:
            scales = [float(scale)] * k
        if not isinstance(start, (list, tuple)) and isinstance(end, (list, tuple)):
            start = [start] * len(end)
        elif not isinstance(end, (list, tuple)) and isinstance(start, (list, tuple)):
            end = [end] * len(start)
        elif not isinstance(start, (list, tuple)) and not isinstance(end, (list, tuple)):
            start, end = [start] * k, [end] * k
        if len(start) != len(end):
            raise ValueError(f"`control_guidance_start` has {len(start)} entries, `control_guidance_end` {len(end)}")
        if len(start) != k:
            raise ValueError(f"`control_guidance_start` / `end` have {len(start)} entries for {k} ControlNets")
        return list(image), scales, [float(s) for s in start], [float(e) for e in end]

    @torch.no_grad()
    def __call__(self, prompt: Optional[Union[str, List[str]]] = None, prompt_2=None, image=None,
                 height: Optional[int] = None, width: Optional[int] = None, num_inference_steps: int = 50,
                 guidance_scale: float = 5.0, negative_prompt=None, negative_prompt_2=None,
                 num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, controlnet_conditioning_scale: float = 1.0,
                 guess_mode: bool = False, control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left=(0, 0), negative_target_size=None, guidance_rescale: float = 0.0,
                 **kwargs):
        """diffusers' parameter list: `image` is the control image (PIL image(s) or a tensor in [0, 1]); height and
        width default to its size floored to multiples of 8.  Unknown keywords are ignored as in the text-to-image
        pipeline, except the arguments in UNSUPPORTED, which raise IHError."""
        from imagharmony_b200.controlnet import ControlNetCall, MultiControlNetModel, controlnet_keep
        self._require_latent_unet()
        self._refuse_unsupported(kwargs)
        multi = isinstance(self.controlnet, MultiControlNetModel)
        if not multi and (isinstance(controlnet_conditioning_scale, (list, tuple))
                          or isinstance(control_guidance_start, (list, tuple))
                          or isinstance(control_guidance_end, (list, tuple))):
            raise IHError("lists of scales / guidance windows need a Multi-ControlNet (a list of ControlNets)")
        if image is None:
            raise ValueError("`image` (the control image) cannot be undefined")
        if multi:
            images, scales, starts, ends = self._align_multi(image, controlnet_conditioning_scale,
                                                             control_guidance_start, control_guidance_end)
        else:
            images, scales = [image], [float(controlnet_conditioning_scale)]
            starts, ends = [control_guidance_start], [control_guidance_end]
        for start, end in zip(starts, ends):                                  # [3P] check_inputs
            if not 0.0 <= start < end <= 1.0:
                raise ValueError(f"control guidance window [{start}, {end}] must satisfy 0 <= start < end <= 1")
        self._check_callback_steps(callback, callback_steps)
        controls = [preprocess_control_image(im, height, width, self.vae_scale_factor) for im in images]
        height, width = controls[0].shape[2], controls[0].shape[3]
        if any(tuple(c.shape[2:]) != (height, width) for c in controls):
            raise ValueError(f"the control images come out at different sizes {[tuple(c.shape[2:]) for c in controls]}; "
                             "pass images of one size, or height and width")
        height, width = self._checked_size(height, width)
        embeds, sizes = self._embeds_and_sizes(locals(), height, width)
        batch = embeds[0].shape[0]
        # [3P] prepare_image, per net: repeat_interleave by the batch (one image) or by num_images_per_prompt; the CFG
        # copy is the engine's (the embedding is computed once and duplicated)
        for j, c in enumerate(controls):
            controls[j] = c.repeat_interleave(batch if c.shape[0] == 1 else (num_images_per_prompt or 1), dim=0)
            if controls[j].shape[0] != batch:
                raise ValueError(f"a control-image batch of {controls[j].shape[0]} does not match the prompt batch of "
                                 f"{batch}")
        self.scheduler.set_timesteps(num_inference_steps)
        lat = self.prepare_latents(batch, self.unet.config.in_channels, height, width, torch.float16, self.device,
                                   generator, latents)
        models = list(self.controlnet.nets) if multi else [self.controlnet]
        cn = [ControlNetCall(m, c.half(), s, bool(guess_mode), controlnet_keep(num_inference_steps, start, end))
              for m, c, s, start, end in zip(models, controls, scales, starts, ends)]
        # the IP scale is not gated: its window stays [0, 1]
        out = self._denoise_from(lat, num_inference_steps=num_inference_steps, embeds=embeds, sizes=sizes,
                                 guidance_scale=guidance_scale, guidance_rescale=guidance_rescale, callback=callback,
                                 callback_steps=callback_steps, generator=generator, controlnet=cn if multi else cn[0])
        return self._output(out, output_type, return_dict)


def preprocess_adapter_image(image, height: int, width: int) -> torch.Tensor:
    """[3P] diffusers' _preprocess_adapter_image (pipeline_stable_diffusion_xl_adapter.py): a tensor is returned as it
    is; PIL image(s) are resized with Lanczos to width x height and divided by 255, a grayscale image giving one channel
    ([h, w] -> [1, 1, h, w], [h, w, c] -> [1, c, h, w]); a list of [C, H, W] tensors is stacked and a list of
    [B, C, H, W] tensors concatenated.  -> float32 [B, C, height, width] (PIL) or the tensor(s) as given."""
    import numpy as np
    from PIL import Image
    if isinstance(image, torch.Tensor):
        return image
    if isinstance(image, Image.Image):
        image = [image]
    if isinstance(image, (list, tuple)) and image and isinstance(image[0], Image.Image):
        arrs = [np.array(im.resize((width, height), resample=Image.LANCZOS)) for im in image]
        arrs = [a[None, ..., None] if a.ndim == 2 else a[None, ...] for a in arrs]
        arr = np.concatenate(arrs, axis=0).astype(np.float32) / 255.0
        return torch.from_numpy(arr.transpose(0, 3, 1, 2).copy())
    if isinstance(image, (list, tuple)) and image and isinstance(image[0], torch.Tensor):
        if image[0].ndim == 3:
            return torch.stack(list(image), dim=0)
        if image[0].ndim == 4:
            return torch.cat(list(image), dim=0)
        raise ValueError(f"Invalid image tensor! Expecting image tensor with 3 or 4 dimension, but recive: "
                         f"{image[0].ndim}")
    raise ValueError(f"the adapter `image` must be a PIL image, a list of them, a tensor or a list of tensors, got "
                     f"{type(image).__name__}")


class StableDiffusionXLAdapterPipeline(StableDiffusionXLCustomPipeline):
    """Text-to-image with an SDXL T2I-Adapter, with the call surface of [3P] diffusers 0.30
    `StableDiffusionXLAdapterPipeline`, so that `IPAdapterXL(adapter_pipe, ...).generate(pil_image=..., image=sketch,
    adapter_conditioning_scale=s)` combines an image prompt with a layout image.  The adapter runs once per call
    (imagharmony_b200.t2i_adapter); its features are added inside the UNet's encoder in the replayed step graph
    (DenoiseEngine.run(adapter=...)) at the steps i < int(num_inference_steps * adapter_conditioning_factor), where
    num_inference_steps counts the steps left after a denoising_end cut.

    `adapter` may be a list of T2IAdapters, wrapped in a MultiAdapter as diffusers does, or a MultiAdapter.  Then
    `image` is a list with one image (or batch) per adapter and `adapter_conditioning_scale` a list of weights (a float
    is taken as the weight of every adapter, an extension: diffusers' MultiAdapter fails on a float); the weighted sum is
    formed once per call.

    As in diffusers, the features are repeated num_images_per_prompt times as a whole ([a, b] -> [a, b, a, b]) and
    then for the CFG halves, and must then equal the prompt batch or, without CFG, be one image; any other image batch
    raises IHError before any work.  One layout image for num_samples > 1 images of IPAdapterXL.generate is therefore
    passed as a list of num_samples copies.

    `control_guidance_start` / `control_guidance_end` gate the IP-adapter scale, as in the text-to-image pipeline.
    T2I-Adapter image-to-image / inpainting / refiner, together with ControlNet or PNS resume, and the SD1.5 adapter
    types are not built (IHError); so are the diffusers arguments in UNSUPPORTED."""

    UNSUPPORTED = ("timesteps", "sigmas", "ip_adapter_image", "ip_adapter_image_embeds", "clip_skip",
                   "callback_on_step_end", "denoising_start")

    def __init__(self, unet: UNet2DConditionModel, adapter, prompt_encoder: Optional[Callable] = None,
                 vae_decode: Optional[Callable] = None, scheduler=None, vae=None):
        from imagharmony_b200.t2i_adapter import MultiAdapter, T2IAdapter
        if isinstance(adapter, (list, tuple)):              # [3P] diffusers wraps a list the same way
            adapter = MultiAdapter(adapter)
        if not isinstance(adapter, (T2IAdapter, MultiAdapter)):
            raise IHError(f"StableDiffusionXLAdapterPipeline: adapter must be a T2IAdapter, a MultiAdapter or a list of "
                          f"T2IAdapters, got {type(adapter).__name__}")
        super().__init__(unet, prompt_encoder=prompt_encoder, vae_decode=vae_decode, scheduler=scheduler, vae=vae)
        self.adapter = adapter

    @classmethod
    def from_random(cls, cfg: UNetConfig = SDXL_BASE, adapter_cfg=None, seed: int = 0, device="cuda", vae_cfg=None):
        """Random-init UNet and adapter weights (SDXL_T2I_ADAPTER by default).  A list of adapter configs gives a
        MultiAdapter pipeline, adapter j seeded with seed + 31 + 7j."""
        from imagharmony_b200.config import SDXL_T2I_ADAPTER
        from imagharmony_b200.t2i_adapter import T2IAdapter
        adapter_cfg = SDXL_T2I_ADAPTER if adapter_cfg is None else adapter_cfg
        base = StableDiffusionXLCustomPipeline.from_random(cfg, seed=seed, device=device, vae_cfg=vae_cfg)
        cfgs = adapter_cfg if isinstance(adapter_cfg, (list, tuple)) else [adapter_cfg]
        ads = [random_module(T2IAdapter, c, seed + 31 + 7 * j, device) for j, c in enumerate(cfgs)]
        return cls(base.unet, ads if isinstance(adapter_cfg, (list, tuple)) else ads[0], vae=base.vae)

    @classmethod
    def from_pretrained(cls, path: str, adapter=None, torch_dtype=torch.float16, add_watermarker: bool = False,
                        device="cuda", cfg: Optional[UNetConfig] = None, vae_cfg=None, **kwargs):
        """`adapter=T2IAdapter.from_pretrained(dir)` (or a list of them, or a MultiAdapter) with the SDXL folder `path`
        of StableDiffusionXLCustomPipeline.from_pretrained; refused before anything is read without it."""
        if adapter is None:
            raise ValueError("StableDiffusionXLAdapterPipeline.from_pretrained needs adapter=")
        return super().from_pretrained(path, torch_dtype, add_watermarker, device, cfg, vae_cfg, adapter=adapter)

    @classmethod
    def _from_parts(cls, parts: _Pretrained, device, adapter=None, **kwargs):
        return cls(parts.unet, adapter, prompt_encoder=parts.prompt_encoder, vae=parts.vae)

    def _default_height_width(self, height: Optional[int], width: Optional[int], image) -> Tuple[int, int]:
        """[3P] diffusers: the first image's size (the first of nested lists), rounded down to a multiple of the
        adapter's downscale factor (16); sizes given are kept."""
        from PIL import Image
        while isinstance(image, list):
            image = image[0]
        f = self.adapter.downscale_factor
        if height is None:
            height = image.height if isinstance(image, Image.Image) else int(image.shape[-2])
            height = (height // f) * f
        if width is None:
            width = image.width if isinstance(image, Image.Image) else int(image.shape[-1])
            width = (width // f) * f
        return height, width

    @torch.no_grad()
    def __call__(self, prompt: Optional[Union[str, List[str]]] = None, prompt_2=None, image=None,
                 height: Optional[int] = None, width: Optional[int] = None, num_inference_steps: int = 50,
                 denoising_end: Optional[float] = None, guidance_scale: float = 5.0, negative_prompt=None,
                 negative_prompt_2=None, num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left=(0, 0), negative_target_size=None,
                 adapter_conditioning_scale: Union[float, List[float]] = 1.0, adapter_conditioning_factor: float = 1.0,
                 control_guidance_start: float = 0.0, control_guidance_end: float = 1.0, **kwargs):
        """diffusers' parameter list: `image` is the adapter image (PIL image(s) or a tensor in [0, 1]; for a
        MultiAdapter one per adapter); height and width default to its size rounded down to a multiple of 16.  Unknown
        keywords are ignored as in the text-to-image pipeline, except the arguments in UNSUPPORTED, which raise
        IHError."""
        from imagharmony_b200.t2i_adapter import AdapterCall, MultiAdapter, adapter_keep, require_image_size
        self._require_latent_unet()
        self._refuse_unsupported(kwargs)
        if image is None:
            raise ValueError("`image` (the adapter image) cannot be undefined")
        multi = isinstance(self.adapter, MultiAdapter)
        if multi:
            k = self.adapter.num_adapter
            if not isinstance(image, list) or len(image) != k:
                raise ValueError(f"MultiAdapter is enabled: `image` must be a list with one entry per adapter ({k})")
            scales = adapter_conditioning_scale
            scales = [float(s) for s in scales] if isinstance(scales, (list, tuple)) else [float(scales)] * k
            if len(scales) != k:
                raise ValueError(f"`adapter_conditioning_scale` has {len(scales)} entries for {k} adapters")
        elif isinstance(adapter_conditioning_scale, (list, tuple)):
            raise IHError("a list of adapter_conditioning_scale values needs a MultiAdapter (a list of adapters)")
        height, width = self._default_height_width(height, width, image)
        inputs = [preprocess_adapter_image(im, height, width) for im in (image if multi else [image])]
        c_in = self.adapter.config.in_channels
        for x in inputs:
            if x.dim() != 4 or x.shape[1] != c_in or tuple(x.shape[2:]) != (height, width):
                raise IHError(f"adapter image {tuple(x.shape)}: expected [B, {c_in}, {height}, {width}] (a tensor is "
                              "not resized; a PIL image's mode must give the adapter's in_channels)")
        if any(x.shape[0] != inputs[0].shape[0] for x in inputs):
            raise IHError(f"MultiAdapter: the adapter images' batches differ: {[x.shape[0] for x in inputs]}")
        height, width = self._checked_size(height, width)
        require_image_size(self.adapter.config, height, width)
        self._check_callback_steps(callback, callback_steps)
        nipp = num_images_per_prompt or 1
        if prompt_embeds is not None:
            batch = prompt_embeds.shape[0]
        elif prompt is not None:
            batch = (1 if isinstance(prompt, str) else len(prompt)) * nipp
        else:
            raise ValueError("Provide either `prompt` or `prompt_embeds`")
        fb = inputs[0].shape[0] * nipp
        if fb != batch and not (guidance_scale <= 1.0 and fb == 1):
            raise IHError(f"an adapter-image batch of {inputs[0].shape[0]} repeated {nipp} times does not broadcast "
                          f"against the prompt batch of {batch} (diffusers adds the features without repeating them "
                          "per prompt: pass one adapter image per prompt)")
        embeds, sizes = self._embeds_and_sizes(locals(), height, width)
        dev = self.device
        self.scheduler.set_timesteps(num_inference_steps)
        lat = self.prepare_latents(batch, self.unet.config.in_channels, height, width, torch.float16, dev,
                                   generator, latents)
        if multi:
            feats = self.adapter([x.to(dev) for x in inputs], scales)
            scale = 1.0
        else:
            feats = self.adapter(inputs[0].to(dev))
            scale = float(adapter_conditioning_scale)
        feats = [f.repeat(nipp, 1, 1, 1) for f in feats]                    # [3P] v.repeat(num_images_per_prompt, ...)
        feats = [f.expand(batch, -1, -1, -1).contiguous() if f.shape[0] != batch else f for f in feats]  # broadcast
        loop_end = self._loop_end(num_inference_steps, denoising_end)
        call = AdapterCall(feats, scale, adapter_keep(num_inference_steps, loop_end, adapter_conditioning_factor))
        out = self._denoise_from(lat, num_inference_steps=num_inference_steps, embeds=embeds, sizes=sizes,
                                 guidance_scale=guidance_scale, guidance_rescale=guidance_rescale,
                                 denoising_end=denoising_end, control_guidance_start=control_guidance_start,
                                 control_guidance_end=control_guidance_end, callback=callback,
                                 callback_steps=callback_steps, generator=generator, adapter=call)
        return self._output(out, output_type, return_dict)
