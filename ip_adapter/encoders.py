"""SDXL prompt conditioning through the two CLIP text encoders, and the CLIP image encoder of the adapter (scope row f2;
[3P] diffusers `encode_prompt` as called at ip_adapter.py:292-297,314-319 / custom_pipelines.py:229-247; image encoder
ip_adapter.py:81-84,163-164).

The towers run on the native kernels (`imagharmony_b200.clip`: wgmma GEMMs with GELU / quick-GELU epilogues, the
generic causal attention kernel, LayerNorm); `transformers` is used for what is host work in the reference too -- the
BPE tokenizers, the PIL image preprocessing and reading a checkpoint folder.  Semantics restated from diffusers==0.30.0:
  * each prompt is tokenised by both tokenizers with padding="max_length" (77) and truncation;
  * prompt_embeds = concat(hidden_states[-2] of encoder 1 [.., 768], hidden_states[-2] of encoder 2 [.., 1280]) -> 2048;
  * pooled_prompt_embeds = `text_embeds` of encoder 2 (the projected pooled output) -> 1280;
  * a model that ships only tokenizer_2 / text_encoder_2 (the SDXL refiner) encodes with tower 2 alone:
    prompt_embeds = its hidden_states[-2] [.., 1280] (encode_prompt with text_encoder = None).
No weights or tokenizer vocabularies exist offline; tests build random CLIP models and a toy vocabulary."""
from __future__ import annotations

import os
from typing import List, Tuple

import torch

from imagharmony_b200.clip import ClipTextTower, ClipVisionTower


class ClipPromptEncoder:
    def __init__(self, tokenizer, tokenizer_2, text_encoder, text_encoder_2, device="cuda", dtype=torch.float16):
        """`text_encoder*`: transformers CLIPTextModel / CLIPTextModelWithProjection instances (their weights are copied
        into native towers and the HF modules are dropped) or ready `ClipTextTower`s.  `tokenizer` and `text_encoder`
        may both be None: the single-tower (refiner) mode."""
        if (tokenizer is None) != (text_encoder is None) or tokenizer_2 is None or text_encoder_2 is None:
            raise ValueError("ClipPromptEncoder needs tokenizer_2 and text_encoder_2, and tokenizer with text_encoder "
                             "(both or neither)")
        pairs = [(tokenizer, text_encoder), (tokenizer_2, text_encoder_2)]
        if text_encoder is None:
            pairs = pairs[1:]
        self.tokenizers = [t for t, _ in pairs]
        self.text_encoders = [e if isinstance(e, ClipTextTower) else ClipTextTower.from_hf(e, device=device)
                              for _, e in pairs]
        self.device, self.dtype = device, dtype

    @classmethod
    def from_pretrained(cls, path: str, device="cuda", dtype=torch.float16) -> "ClipPromptEncoder":
        """`path` = an SDXL snapshot folder with tokenizer_2/ and text_encoder_2/, and tokenizer/ and text_encoder/
        unless it is a single-tower model (the refiner)."""
        from transformers import CLIPTextModel, CLIPTextModelWithProjection, CLIPTokenizer
        one = not cls._has(path, ("tokenizer", "text_encoder"))
        return cls(None if one else CLIPTokenizer.from_pretrained(os.path.join(path, "tokenizer")),
                   CLIPTokenizer.from_pretrained(os.path.join(path, "tokenizer_2")),
                   None if one else CLIPTextModel.from_pretrained(os.path.join(path, "text_encoder")),
                   CLIPTextModelWithProjection.from_pretrained(os.path.join(path, "text_encoder_2")), device, dtype)

    @staticmethod
    def _has(path: str, dirs) -> bool:
        return all(os.path.isdir(os.path.join(path, d)) for d in dirs)

    @staticmethod
    def available(path: str) -> bool:
        return ClipPromptEncoder._has(path, ("tokenizer_2", "text_encoder_2"))

    @torch.no_grad()
    def __call__(self, prompts: List[str]) -> Tuple[torch.Tensor, torch.Tensor]:
        embeds, pooled = [], None
        for tok, enc in zip(self.tokenizers, self.text_encoders):
            ids = tok(list(prompts), padding="max_length", max_length=tok.model_max_length, truncation=True,
                      return_tensors="pt").input_ids
            out = enc(ids, output_hidden_states=True)
            # [3P] encode_prompt keeps `prompt_embeds[0]` of the LAST encoder only: its projected `text_embeds`
            pooled = out.text_embeds if out.text_embeds is not None else out.pooler_output
            embeds.append(out.penultimate)             # penultimate layer (clip_skip = None)
        return torch.cat(embeds, dim=-1).to(torch.float16), pooled.to(torch.float16)


def load_image_encoder(path: str, device="cuda") -> ClipVisionTower:
    """ip_adapter.py:81-83: CLIPVisionModelWithProjection.from_pretrained(path) -> native vision tower."""
    from transformers import CLIPVisionModelWithProjection
    return ClipVisionTower.from_hf(CLIPVisionModelWithProjection.from_pretrained(path), device=device)
