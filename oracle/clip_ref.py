"""ORACLE (test infrastructure only) for scope row f2.

The CLIP towers' arithmetic lives in `transformers` ([3P], requirements.txt:145 pins 4.45.0; 5.5.0 is installed in this
image and on the GPU box): the oracle for `imagharmony_b200.clip` IS that library -- `hf_text_model` / `hf_vision_model`
build random-init `CLIPTextModel(WithProjection)` / `CLIPVisionModelWithProjection` instances whose fp32 CPU forward the
tests compare against (reference call sites: ip_adapter.py:81-84,163-164,404-412; encode_prompt :292-319).
`resize_patchify_ref` restates the scorer's device-side preprocessing (area-average resize, CLIP normalisation, patch
rows) in plain PyTorch.
"""
from __future__ import annotations

import torch

# shapes of the real towers ([3P] model cards): SDXL text_encoder (CLIP ViT-L/14 text), text_encoder_2 (OpenCLIP bigG
# text), IP-Adapter SDXL image encoder (OpenCLIP ViT-bigG/14), IP-Adapter "vit-h" image encoder (ViT-H/14)
TEXT_L = dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
              hidden_act="quick_gelu", projection_dim=768)
TEXT_BIGG = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=20,
                 hidden_act="gelu", projection_dim=1280)
VISION_BIGG = dict(hidden_size=1664, intermediate_size=8192, num_hidden_layers=48, num_attention_heads=16,
                   hidden_act="gelu", projection_dim=1280, image_size=224, patch_size=14)
VISION_H = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16,
                hidden_act="gelu", projection_dim=1024, image_size=224, patch_size=14)


def hf_text_model(seed: int, with_projection: bool, vocab_size: int = 49408, eos_token_id: int = 49407, **kw):
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    torch.manual_seed(seed)
    cfg = CLIPTextConfig(vocab_size=vocab_size, max_position_embeddings=77, bos_token_id=vocab_size - 2,
                         eos_token_id=eos_token_id, pad_token_id=eos_token_id, **kw)
    m = (CLIPTextModelWithProjection if with_projection else CLIPTextModel)(cfg)
    return _fp16_representable(m).eval()


def hf_vision_model(seed: int, **kw):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    torch.manual_seed(seed)
    return _fp16_representable(CLIPVisionModelWithProjection(CLIPVisionConfig(**kw))).eval()


def _fp16_representable(m):
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(p.half().float())
    return m


def resize_patchify_ref(img: torch.Tensor, size: int, patch: int, kpad: int, mean, std,
                        dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """img [B, 3, H, W] in [-1, 1] on the CPU -> area-average to size x size (exact box filter with fractional pixel
    coverage) -> [0, 1] clamp -> (v - mean) / std -> patch rows [B * (size/patch)^2, kpad], k = c*P*P + py*P + px,
    computed in `dtype` (fp32; fp64 for the per-call kernel census)."""
    B, C, H, W = img.shape

    def weights(n_in: int) -> torch.Tensor:          # [size, n_in] coverage of input pixel x by output pixel o
        f = n_in / size
        o = torch.arange(size, dtype=torch.float64)[:, None]
        x = torch.arange(n_in, dtype=torch.float64)[None, :]
        w = (torch.minimum((o + 1) * f, x + 1) - torch.maximum(o * f, x)).clamp_min(0)
        return (w / w.sum(dim=1, keepdim=True)).to(dtype)
    wy, wx = weights(H), weights(W)
    small = torch.einsum("oy,bcyx,px->bcop", wy, img.to(dtype), wx)
    v = (small * 0.5 + 0.5).clamp(0, 1)
    v = (v - torch.tensor(mean, dtype=dtype).view(1, 3, 1, 1)) / torch.tensor(std, dtype=dtype).view(1, 3, 1, 1)
    g = size // patch
    rows = v.reshape(B, C, g, patch, g, patch).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, C * patch * patch)
    out = torch.zeros((B * g * g, kpad), dtype=dtype)
    out[:, : rows.shape[1]] = rows
    return out
