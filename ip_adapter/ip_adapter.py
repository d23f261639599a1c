"""IPAdapter / IPAdapterXL / IPAdapterPlusXL with the reference's constructor and method surface
(reference ip_adapter/ip_adapter.py:69-340, 389-478) driving the native pipeline.

What is preserved: argument names/defaults, attribute names (.pipe, .image_encoder, .clip_image_processor,
.image_proj_model, .number_class_crossattention, .device, .num_tokens, .generator), set_ip_adapter's layer selection
(IP branch only where the processor name contains 'down_blocks.2.attentions.1', :117; `target_blocks` is accepted and
ignored exactly like the reference, :75), the 3-key checkpoint layout of load_ip_adapter (:149-154), get_image_embeds,
set_scale and generate().

Positions taken on reference quirks (SURVEY.md appendix C): `extra_text=None` skips the HarmonyAttention residual
instead of raising NameError (C.5); the .safetensors branch is implemented correctly instead of KeyError-ing (C.6);
the forward-time prints of HarmonyAttention are dropped (C.10); one copy of the auxiliary text feeds HA (C.11).
"""
from __future__ import annotations

import os

import torch
from PIL import Image

from imagharmony_b200._lib import IHError
from imagharmony_b200.adapter import HarmonyAttention, ImageProjModel, Resampler  # noqa: F401
from imagharmony_b200.controlnet import MultiControlNetModel
from imagharmony_b200.taesd import AutoencoderTiny  # noqa: F401  (re-exported: pipe.vae = AutoencoderTiny.from_pretrained)

from .utils import get_generator, is_torch2_available

if is_torch2_available():
    from .attention_processor import AttnProcessor2_0 as AttnProcessor
    from .attention_processor import CNAttnProcessor2_0 as CNAttnProcessor
    from .attention_processor import IPAttnProcessor2_0 as IPAttnProcessor
else:  # pragma: no cover
    from .attention_processor import AttnProcessor, CNAttnProcessor, IPAttnProcessor


DEFAULT_PROMPT = "best quality, high quality"                                           # reference :276, :441
DEFAULT_NEGATIVE_PROMPT = "monochrome, lowres, bad anatomy, worst quality, low quality"     # reference :278, :443
IP_LAYER_MARKER = "down_blocks.2.attentions.1"   # the only attn2 layers whose IP branch is active (reference :117)

# prefixes under which the three parts of an adapter checkpoint appear in a flat (.safetensors / accelerate) file
_CKPT_PREFIXES = (("image_proj.", "image_proj"), ("image_proj_model.", "image_proj"), ("ip_adapter.", "ip_adapter"),
                  ("adapter_modules.", "ip_adapter"), ("composed_adapter.", "composed_adapter"),
                  ("composed_modules.", "composed_adapter"))


def _block_channels(proc_name: str, channels) -> int:
    """Width of the attention module a processor name belongs to (`<down|up>_blocks.<i>...` / `mid_block...`)."""
    head, _, rest = proc_name.partition(".")
    if head == "mid_block":
        return channels[-1]
    level = int(rest.split(".", 1)[0])
    if head == "up_blocks":
        return channels[len(channels) - 1 - level]
    if head == "down_blocks":
        return channels[level]
    raise IHError(f"unexpected attention processor name {proc_name!r}")


def _per_image(value, default, count):
    """prompt / negative_prompt argument -> one string per input image"""
    value = default if value is None else value
    return list(value) if isinstance(value, (list, tuple)) else [value] * count


def _repeat_for_samples(t: torch.Tensor, num_samples: int) -> torch.Tensor:
    """[b, n, d] -> [b * num_samples, n, d], the copies of one image adjacent (reference :302-306)"""
    b, n, d = t.shape
    return t.unsqueeze(1).expand(b, num_samples, n, d).reshape(b * num_samples, n, d)


class IPAdapter:
    def __init__(self, sd_pipe, image_encoder_path, ip_ckpt, device, num_tokens=4, target_blocks=None,
                 number_class_crossattention=None):
        if sd_pipe.unet.config.num_ip_tokens == 0:
            raise IHError("this UNet has no image-prompt layers (num_ip_tokens = 0, e.g. the SDXL refiner): the "
                          "IMAGHarmony adapter is trained for the SDXL base UNet")
        self.device, self.num_tokens = device, num_tokens
        self.image_encoder_path, self.ip_ckpt = image_encoder_path, ip_ckpt
        self.pipe = sd_pipe.to(device)
        self.set_ip_adapter()

        # image encoder (CLIP ViT-bigG/14 with projection for SDXL, reference :81-84): the checkpoint folder is read with
        # transformers, the tower itself runs on the native kernels (imagharmony_b200.clip.ClipVisionTower, row f2).
        # `image_encoder_path` may also be a ready ClipVisionTower (tests: no weights exist offline).
        self.image_encoder = None
        self.clip_image_processor = None
        from imagharmony_b200.clip import ClipVisionTower
        if isinstance(image_encoder_path, ClipVisionTower):
            self.image_encoder = image_encoder_path
        elif image_encoder_path is not None and os.path.isdir(str(image_encoder_path)):
            from .encoders import load_image_encoder
            self.image_encoder = load_image_encoder(image_encoder_path, self.device)
        if self.image_encoder is not None:
            from transformers import CLIPImageProcessor
            self.clip_image_processor = CLIPImageProcessor()
        self.number_class_crossattention = None
        if number_class_crossattention is not None:
            self.number_class_crossattention = number_class_crossattention.to(self.device, dtype=torch.float16)
        self.image_proj_model = self.init_proj()
        self.generator = None
        self.load_ip_adapter()

    # ---- reference :91-97 -------------------------------------------------------------------------------------------
    def _clip_dim(self) -> int:
        if self.image_encoder is not None:
            return self.image_encoder.config.projection_dim
        if self.number_class_crossattention is not None:
            return self.number_class_crossattention.image_hidden_size
        return self.pipe.unet.config.pooled_embed_dim

    def init_proj(self):
        proj = ImageProjModel(cross_attention_dim=self.pipe.unet.config.cross_attention_dim,
                              clip_embeddings_dim=self._clip_dim(), clip_extra_context_tokens=self.num_tokens)
        return proj.to(self.device, dtype=torch.float16).requires_grad_(False)

    # ---- reference :99-133 ------------------------------------------------------------------------------------------
    def set_ip_adapter(self):
        """One processor per attention module: plain for self-attention, decoupled image-prompt processors for the 70
        cross-attention modules -- with the image branch switched on only inside IP_LAYER_MARKER.  On a ControlNet
        pipeline the ControlNet gets CNAttnProcessor (reference :128-133): it sees the text tokens only."""
        cfg = self.pipe.unet.config
        table = {}
        for name in self.pipe.unet.attn_processors:
            if name.endswith("attn1.processor"):
                table[name] = AttnProcessor()
                continue
            with torch.device("meta"):
                proc = IPAttnProcessor(hidden_size=_block_channels(name, cfg.block_out_channels),
                                       cross_attention_dim=cfg.cross_attention_dim, num_tokens=self.num_tokens,
                                       skip=IP_LAYER_MARKER not in name)
            proc = proc.to_empty(device=self.device).to(torch.float16).requires_grad_(False)
            for prm in proc.parameters():
                prm.zero_()                       # inert until load_ip_adapter fills to_k_ip / to_v_ip
            table[name] = proc
        self.pipe.unet.set_attn_processor(table)
        if hasattr(self.pipe, "controlnet"):
            if isinstance(self.pipe.controlnet, MultiControlNetModel):
                for controlnet in self.pipe.controlnet.nets:
                    controlnet.set_attn_processor(CNAttnProcessor(num_tokens=self.num_tokens))
            else:
                self.pipe.controlnet.set_attn_processor(CNAttnProcessor(num_tokens=self.num_tokens))

    # ---- reference :135-154 -----------------------------------------------------------------------------------------
    def load_ip_adapter(self):
        if self.ip_ckpt is None:
            return   # random / zero-initialised adapter (benchmarks and tests: there are no checkpoints offline)
        if str(self.ip_ckpt).endswith(".safetensors"):
            from safetensors import safe_open
            parts = {"image_proj": {}, "ip_adapter": {}, "composed_adapter": {}}
            with safe_open(self.ip_ckpt, framework="pt", device="cpu") as fh:
                for key in fh.keys():
                    hit = next(((pre, dst) for pre, dst in _CKPT_PREFIXES if key.startswith(pre)), None)
                    if hit is not None:
                        parts[hit[1]][key[len(hit[0]):]] = fh.get_tensor(key)
        else:
            parts = torch.load(self.ip_ckpt, map_location="cpu")                   # the 3-key dict of convert_bin.py
        self.image_proj_model.load_state_dict(parts["image_proj"])
        if self.number_class_crossattention is not None:
            if not parts.get("composed_adapter"):
                # the reference loads this part strictly (:151-152): a HarmonyAttention module without its weights would
                # add a residual from random parameters to every image embedding
                raise KeyError("composed_adapter: number_class_crossattention was given but the checkpoint holds no "
                               "HarmonyAttention weights")
            self.number_class_crossattention.load_state_dict(parts["composed_adapter"])
        # strict and index-keyed: every one of the 70 cross-attention processors owns to_k_ip / to_v_ip (:153)
        torch.nn.ModuleList(self.pipe.unet.attn_processors.values()).load_state_dict(parts["ip_adapter"])
        self.pipe.unet.finalize()

    # ---- reference :158-182 -----------------------------------------------------------------------------------------
    @torch.inference_mode()
    def get_image_embeds(self, pil_image=None, clip_image_embeds=None, extra_prompt_embeds=None):
        """-> (conditional, unconditional) image-prompt tokens [n, num_tokens, cross_attention_dim]."""
        if pil_image is None:
            emb = clip_image_embeds
        else:
            if self.image_encoder is None:
                raise IHError("no CLIP image encoder loaded (image_encoder_path): pass clip_image_embeds=")
            images = [pil_image] if isinstance(pil_image, Image.Image) else list(pil_image)
            pixels = self.clip_image_processor(images=images, return_tensors="pt").pixel_values
            emb = self.image_encoder(pixels).image_embeds
        emb = emb.to(self.device, dtype=torch.float16).contiguous()
        if extra_prompt_embeds is not None and self.number_class_crossattention is not None:      # :169-173
            aux = extra_prompt_embeds.to(self.device, torch.float16)
            emb = self.number_class_crossattention(aux, emb, add_to=emb)      # harmony-aware residual on the embedding
        return self.image_proj_model(emb), self.image_proj_model(torch.zeros_like(emb))           # :175-176

    def set_scale(self, scale):
        for proc in self.pipe.unet.attn_processors.values():
            if isinstance(proc, IPAttnProcessor):
                proc.scale = scale


class IPAdapterXL(IPAdapter):
    """SDXL"""

    def __init__(self, sd_pipe, image_encoder_path, ip_ckpt, device, num_tokens=4, target_blocks=None,
                 inference=False, number_class_crossattention=None):
        self.inference = inference
        super().__init__(sd_pipe, image_encoder_path, ip_ckpt, device, num_tokens=num_tokens,
                         target_blocks=target_blocks, number_class_crossattention=number_class_crossattention)

    def generate(self, pil_image=None, prompt=None, negative_prompt=None, extra_text=None, scale=1.0, num_samples=4,
                 seed=None, num_inference_steps=30, clip_image_embeds=None, **kwargs):
        """reference :257-340.  `clip_image_embeds=` is an extension for environments without the CLIP vision weights."""
        self.set_scale(scale)
        if pil_image is None:
            n_img = clip_image_embeds.shape[0]
        else:
            n_img = 1 if isinstance(pil_image, Image.Image) else len(pil_image)
        prompts = _per_image(prompt, DEFAULT_PROMPT, n_img)
        negatives = _per_image(negative_prompt, DEFAULT_NEGATIVE_PROMPT, n_img)
        cfg_args = dict(num_images_per_prompt=num_samples, do_classifier_free_guidance=True, negative_prompt=negatives)

        aux_embeds = None
        if extra_text is not None:                                                 # :285-297 (auxiliary count/class text)
            aux_embeds = self.pipe.encode_prompt(extra_text, **cfg_args)[0]
        cond, uncond = self.get_image_embeds(pil_image=pil_image, clip_image_embeds=clip_image_embeds,
                                             extra_prompt_embeds=aux_embeds)                       # :300
        cond, uncond = _repeat_for_samples(cond, num_samples), _repeat_for_samples(uncond, num_samples)

        text, neg_text, pooled, neg_pooled = self.pipe.encode_prompt(prompts, **cfg_args)          # :308-319
        prompt_embeds = torch.cat([text.to(cond.device), cond], dim=1)                             # :321 -> 77 + 4 tokens
        negative_prompt_embeds = torch.cat([neg_text.to(cond.device), uncond], dim=1)              # :322

        # a list of seeds means one CPU generator per image, so a candidate noise does not depend on its batch slot
        self.generator = get_generator(seed, "cpu" if isinstance(seed, list) else self.device)     # :328
        result = self.pipe(prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                           pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=neg_pooled,
                           num_inference_steps=num_inference_steps, generator=self.generator, **kwargs)
        return result.images


class IPAdapterPlusXL(IPAdapter):
    """SDXL with the Resampler projector (reference :389-478): 16 image tokens from the CLIP penultimate hidden
    states."""

    def init_proj(self):
        width = self.image_encoder.config.hidden_size if self.image_encoder is not None else 1664   # ViT-bigG
        resampler = Resampler(dim=1280, depth=4, dim_head=64, heads=20, num_queries=self.num_tokens, embedding_dim=width,
                              output_dim=self.pipe.unet.config.cross_attention_dim, ff_mult=4)
        return resampler.to(self.device, dtype=torch.float16).requires_grad_(False)

    @torch.inference_mode()
    def get_image_embeds(self, pil_image=None, clip_hidden_states=None, uncond_clip_hidden_states=None):
        """Resampler tokens of the penultimate CLIP hidden states; the unconditional branch encodes a black image."""
        if pil_image is not None:
            if self.image_encoder is None:
                raise IHError("no CLIP image encoder loaded: pass clip_hidden_states= / uncond_clip_hidden_states=")
            images = [pil_image] if isinstance(pil_image, Image.Image) else list(pil_image)
            pixels = self.clip_image_processor(images=images, return_tensors="pt").pixel_values

            def penultimate(x):
                return self.image_encoder(x, output_hidden_states=True).hidden_states[-2]
            clip_hidden_states, uncond_clip_hidden_states = penultimate(pixels), penultimate(torch.zeros_like(pixels))
        to_dev = lambda t: t.to(self.device, torch.float16)  # noqa: E731
        return self.image_proj_model(to_dev(clip_hidden_states)), self.image_proj_model(to_dev(uncond_clip_hidden_states))

    def generate(self, pil_image=None, prompt=None, negative_prompt=None, scale=1.0, num_samples=4, seed=None,
                 num_inference_steps=30, clip_hidden_states=None, uncond_clip_hidden_states=None, **kwargs):
        """reference :423-478 (no auxiliary text / HarmonyAttention on this variant)."""
        self.set_scale(scale)
        n_img = 1 if (pil_image is None or isinstance(pil_image, Image.Image)) else len(pil_image)
        prompts = _per_image(prompt, DEFAULT_PROMPT, n_img)
        negatives = _per_image(negative_prompt, DEFAULT_NEGATIVE_PROMPT, n_img)
        cond, uncond = self.get_image_embeds(pil_image, clip_hidden_states, uncond_clip_hidden_states)
        cond, uncond = _repeat_for_samples(cond, num_samples), _repeat_for_samples(uncond, num_samples)
        text, neg_text, pooled, neg_pooled = self.pipe.encode_prompt(
            prompts, num_images_per_prompt=num_samples, do_classifier_free_guidance=True, negative_prompt=negatives)
        generator = get_generator(seed, "cpu" if isinstance(seed, list) else self.device)
        return self.pipe(prompt_embeds=torch.cat([text.to(cond.device), cond], dim=1),
                         negative_prompt_embeds=torch.cat([neg_text.to(cond.device), uncond], dim=1),
                         pooled_prompt_embeds=pooled, negative_pooled_prompt_embeds=neg_pooled,
                         num_inference_steps=num_inference_steps, generator=generator, **kwargs).images
