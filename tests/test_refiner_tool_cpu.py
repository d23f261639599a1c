"""Host logic of tools/bench_refiner.py: the UNet FLOP count it reports the refiner's achieved rate with, checked against
torch's FLOP counter on the oracle forward (tests/refiner_ref.py) minus the time embeddings, which the count leaves
out."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_refiner import unet_flops  # noqa: E402


def _time_embedding_flops(cfg, batch):
    T = cfg.time_embed_dim
    from imagharmony_b200.unet import ResnetBlock2D, UNet2DConditionModel
    with torch.device("meta"):
        m = UNet2DConditionModel(cfg)
    couts = sum(r.cout for r in m.modules() if isinstance(r, ResnetBlock2D))
    return batch * (2 * cfg.block_out_channels[0] * T + 2 * T * T + 2 * cfg.add_embed_in * T + 2 * T * T + 2 * T * couts)


@pytest.mark.parametrize("lat", [16, 8])
def test_unet_flops_match_torch_flop_counter(lat):
    from torch.utils.flop_counter import FlopCounterMode
    from imagharmony_b200.config import TINY_REFINER as cfg
    from refiner_ref import unet_ref
    torch.manual_seed(0)
    ref = unet_ref(cfg)
    B = 2
    ids = [128.0] * cfg.num_time_ids
    with FlopCounterMode(display=False) as fc, torch.no_grad():
        ref(torch.randn(B, 4, lat, lat), 500.0, torch.randn(B, 77 + cfg.num_ip_tokens, cfg.cross_attention_dim),
            torch.randn(B, cfg.pooled_embed_dim), torch.tensor([ids] * B))
    assert unet_flops(cfg, 8 * lat, 8 * lat, B) == fc.get_total_flops() - _time_embedding_flops(cfg, B)


def test_refiner_flops_at_1024():
    from imagharmony_b200.config import SDXL_REFINER
    f = unet_flops(SDXL_REFINER, 1024, 1024)
    assert unet_flops(SDXL_REFINER, 1024, 1024, batch=2) == 2 * f
    assert 6.0e12 < f < 8.0e12                       # about 7.3 TFLOP per image at 1024^2
