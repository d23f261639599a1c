"""Deterministic random-init weights (there is no network for checkpoints) and checkpoint-format helpers.

`random_state_dict` fills a {key: shape} description with fp16 values drawn from one seeded generator in key order:
matrices/convs ~ U(-1/sqrt(fan_in), 1/sqrt(fan_in)) (PyTorch's default Linear/Conv bound), biases likewise, norm
weights 1 + 0.1 N(0,1), norm biases 0.1 N(0,1) so the affine paths are exercised.  The oracle loads the same dict
cast to fp32, so both sides see bit-identical (fp16-representable) parameters.  `random_module` builds a native model
from such a dict.

`split_ip_adapter_checkpoint` / `join_ip_adapter_checkpoint` mirror the 3-key layout written by the reference's
convert_bin.py:21-40 ({"image_proj", "ip_adapter", "composed_adapter"}) that ip_adapter.py:149-154 loads.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, Mapping, Tuple

import torch


def shapes_of(module: torch.nn.Module) -> Dict[str, Tuple[int, ...]]:
    return {k: tuple(v.shape) for k, v in module.state_dict().items()}


def random_state_dict(shapes: Mapping[str, Iterable[int]], seed: int = 0, device: str = "cpu",
                      dtype: torch.dtype = torch.float16) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device=device).manual_seed(seed)
    out: Dict[str, torch.Tensor] = {}
    fan_in_of: Dict[str, int] = {}
    norm_prefixes = set()          # modules whose weight is 1-D are normalisation layers
    for key, shape in shapes.items():
        shape = tuple(shape)
        if key.endswith(".weight") and len(shape) >= 2:
            fan_in_of[key[: -len(".weight")]] = int(math.prod(shape[1:]))
        elif key.endswith(".weight") and len(shape) == 1:
            norm_prefixes.add(key[: -len(".weight")])
    for key, shape in shapes.items():
        shape = tuple(shape)
        prefix, _, leaf = key.rpartition(".")
        if prefix in norm_prefixes and len(shape) == 1:
            t = torch.randn(shape, generator=g, device=device, dtype=torch.float32) * 0.1
            if leaf == "weight":
                t = t + 1.0
        elif leaf == "latents":  # Resampler.latents ~ N(0,1)/sqrt(dim) (resampler.py:99)
            t = torch.randn(shape, generator=g, device=device, dtype=torch.float32) / math.sqrt(shape[-1])
        else:
            fan_in = fan_in_of.get(prefix)
            if fan_in is None:
                fan_in = int(math.prod(shape[1:])) if len(shape) >= 2 else max(int(shape[0]), 1)
            bound = 1.0 / math.sqrt(max(fan_in, 1))
            t = (torch.rand(shape, generator=g, device=device, dtype=torch.float32) * 2.0 - 1.0) * bound
        out[key] = t.to(dtype)
    return out


def random_module(cls, cfg, seed: int, device="cuda"):
    """`cls.from_state_dict(cfg, ...)` with random_state_dict(seed) weights for the shapes of `cls(cfg)` (built on the
    meta device), drawn on `device` when it is a CUDA device and on the CPU otherwise."""
    with torch.device("meta"):
        shapes = shapes_of(cls(cfg))
    gen_dev = device if str(device).startswith("cuda") else "cpu"
    return cls.from_state_dict(cfg, random_state_dict(shapes, seed, device=gen_dev), device=device)


def split_ip_adapter_checkpoint(full: Mapping[str, torch.Tensor]) -> Dict[str, Dict[str, torch.Tensor]]:
    """accelerate-style flat dict with prefixes image_proj_model./adapter_modules./composed_modules. -> 3-key dict
    (convert_bin.py:21-40)."""
    out = {"image_proj": {}, "ip_adapter": {}, "composed_adapter": {}}
    for k, v in full.items():
        if k.startswith("image_proj_model."):
            out["image_proj"][k[len("image_proj_model."):]] = v
        elif k.startswith("adapter_modules."):
            out["ip_adapter"][k[len("adapter_modules."):]] = v
        elif k.startswith("composed_modules."):
            out["composed_adapter"][k[len("composed_modules."):]] = v
    return out


def infer_harmony_dims(composed: Mapping[str, torch.Tensor]) -> Dict[str, int]:
    """HarmonyAttention hyper-parameters are not stored in the checkpoint (test.py:9-15 re-types them by hand);
    recover them from tensor shapes (SURVEY.md appendix C.12)."""
    inter_dim, image_hidden = composed["fc1.weight"].shape
    q_dim = composed["fusion_text_image.to_q.weight"].shape[1]
    blocks = inter_dim // q_dim
    v_rows, text_dim = composed["fusion_text_image.to_v.weight"].shape
    flat = composed["ln.weight"].shape[0]
    heads_times_v = flat // blocks
    assert heads_times_v == v_rows
    return {"image_hidden_size": int(image_hidden), "text_context_dim": int(text_dim), "inter_dim": int(inter_dim),
            "reshape_blocks": int(blocks), "heads_times_value_dim": int(heads_times_v), "query_dim": int(q_dim)}
