"""TEST-ONLY restatement of [3P] diffusers 0.30.0 T2IAdapter (adapter_type "full_adapter_xl"), MultiAdapter, the
down_intrablock_additional_residuals of UNet2DConditionModel and StableDiffusionXLAdapterPipeline's feature handling
and loop, fp32 on the CPU by default, built on the oracle's UNet blocks (oracle/unet_ref.py).  It keeps diffusers'
form: nn.PixelUnshuffle, nn.AvgPool2d(2, ceil_mode=True) followed by the separate 1x1 in_conv, NCHW activations,
in-place `sample +=` for the blocks without cross-attention."""
from typing import Callable, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.unet_ref import UNetRef


class AdapterResnetBlockRef(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.block1 = nn.Conv2d(ch, ch, 3, padding=1)
        self.act = nn.ReLU()
        self.block2 = nn.Conv2d(ch, ch, 1)

    def forward(self, x):
        return self.block2(self.act(self.block1(x))) + x


class AdapterBlockRef(nn.Module):
    def __init__(self, cin, cout, num_res_blocks, down=False):
        super().__init__()
        self.downsample = nn.AvgPool2d(kernel_size=2, stride=2, ceil_mode=True) if down else None
        self.in_conv = nn.Conv2d(cin, cout, kernel_size=1) if cin != cout else None
        self.resnets = nn.Sequential(*[AdapterResnetBlockRef(cout) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.downsample is not None:
            x = self.downsample(x)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class FullAdapterXLRef(nn.Module):
    def __init__(self, in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=16):
        super().__init__()
        self.unshuffle = nn.PixelUnshuffle(downscale_factor)
        self.conv_in = nn.Conv2d(in_channels * downscale_factor ** 2, channels[0], kernel_size=3, padding=1)
        body = []
        for i in range(len(channels)):
            if i == 1:
                body.append(AdapterBlockRef(channels[i - 1], channels[i], num_res_blocks))
            elif i == 2:
                body.append(AdapterBlockRef(channels[i - 1], channels[i], num_res_blocks, down=True))
            else:
                body.append(AdapterBlockRef(channels[i], channels[i], num_res_blocks))
        self.body = nn.ModuleList(body)

    def forward(self, x):
        x = self.conv_in(self.unshuffle(x))
        features = []
        for block in self.body:
            x = block(x)
            features.append(x)
        return features


class T2IAdapterRef(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.adapter = FullAdapterXLRef(cfg.in_channels, cfg.channels, cfg.num_res_blocks, cfg.downscale_factor)

    def forward(self, x):
        return self.adapter(x)


def multi_adapter_ref(adapters, xs, adapter_weights=None) -> List[torch.Tensor]:
    """[3P] MultiAdapter.forward: w_0 * f_0, then += w_j * f_j in adapter order, the weights a float32 tensor."""
    n = len(adapters)
    w = torch.tensor([1 / n] * n) if adapter_weights is None else torch.tensor(adapter_weights)
    acc = None
    for x, wj, adapter in zip(xs, w, adapters):
        features = adapter(x)
        if acc is None:
            acc = [wj * f for f in features]
        else:
            for i in range(len(features)):
                acc[i] += wj * features[i]
    return acc


class UNetAdapterRef(UNetRef):
    """UNetRef whose forward also takes down_intrablock_additional_residuals (a list, consumed front to back as in
    diffusers): for a down block without cross-attention `sample += r` after the block (in place: its last skip is
    that tensor), for one with it `hidden_states = hidden_states + r` after the last resnet / attention pair, before
    the skip is appended; a leftover residual with the mid output's shape is added after the mid block."""

    def forward(self, sample, timestep, encoder_hidden_states, text_embeds, time_ids,
                down_intrablock_additional_residuals=None):
        args = (sample, timestep, encoder_hidden_states, text_embeds, time_ids)
        if down_intrablock_additional_residuals is None:
            return super().forward(*args)
        pending = list(down_intrablock_additional_residuals)
        saved = []

        def wrap_plain(blk):
            orig = blk.forward

            def fwd(x, emb, ehs, skips):
                x = orig(x, emb, ehs, skips)
                if pending:
                    x += pending.pop(0)
                return x
            return fwd

        def wrap_attn(blk):
            def fwd(x, emb, ehs, skips):
                r = pending.pop(0) if pending else None
                n = len(blk.resnets)
                for j, res in enumerate(blk.resnets):
                    x = blk.attentions[j](res(x, emb), ehs)
                    if j == n - 1 and r is not None:
                        x = x + r
                    skips.append(x)
                if blk.downsamplers is not None:
                    x = blk.downsamplers[0](x)
                    skips.append(x)
                return x
            return fwd

        for blk in self.down_blocks:
            saved.append(blk)
            blk.forward = wrap_attn(blk) if blk.attentions is not None else wrap_plain(blk)
        mid_fwd = self.mid_block.forward

        def mid(x, emb, ehs):
            x = mid_fwd(x, emb, ehs)
            if pending and x.shape == pending[0].shape:
                x += pending.pop(0)
            return x
        self.mid_block.forward = mid
        try:
            return super().forward(*args)
        finally:
            for blk in saved:
                del blk.forward
            del self.mid_block.forward


def adapter_state_ref(features, conditioning_scale, num_images_per_prompt: int, cfg: bool, multi: bool = False):
    """[3P] the pipeline's features: scaled once (a single adapter; a MultiAdapter's are already weighted), repeated
    num_images_per_prompt times as a whole, then for the CFG halves."""
    state = [v if multi else v * conditioning_scale for v in features]
    if num_images_per_prompt > 1:
        state = [v.repeat(num_images_per_prompt, 1, 1, 1) for v in state]
    if cfg:
        state = [torch.cat([v] * 2, dim=0) for v in state]
    return state


def adapter_unet_fn(unet: UNetAdapterRef, state, loop_steps: int, conditioning_factor: float) -> Callable:
    """unet_fn for the oracle / tests' denoise loops: call i passes clones of the features iff
    i < int(loop_steps * conditioning_factor), loop_steps counted after the denoising_end cut."""
    count = [0]
    active = int(loop_steps * conditioning_factor)

    def fn(sample, t, ehs, te, tids):
        i = count[0]
        count[0] += 1
        res = [s.clone() for s in state] if i < active else None
        return unet(sample, t, ehs, te, tids, down_intrablock_additional_residuals=res)
    return fn


def fold_pool_conv_ref(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor]) -> torch.Tensor:
    """AvgPool2d(2) then a 1x1 conv, as the 2x2-window stride-2 conv the native adapter runs (NCHW, fp32)."""
    w2 = (w / 4).expand(-1, -1, 2, 2)
    return F.conv2d(x, w2, b, stride=2)
