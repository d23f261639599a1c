"""TEST-ONLY stand-ins for the image-to-image ops of imagharmony_b200.ops (conv3x3_down, vae_posterior_noise) in plain
PyTorch on the CPU, used next to tests/fake_ops.py by the image-to-image CPU wiring tests.  Never imported by the
product."""
import torch.nn.functional as F

import fake_ops
from img2img_ref import posterior_noise_ref


def conv3x3_down(x, w_packed, bias=None, *, out=None, tile_n=0, alpha=1.0):
    fake_ops._count[0] += 1
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    w = w_packed.reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2).float()
    y = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w, None, stride=2).permute(0, 2, 3, 1) * alpha
    if bias is not None:
        y = y + bias.float()
    return y.to(x.dtype).contiguous()


def vae_posterior_noise(moments, eps, noise, channels, scaling_factor, sigma, out=None):
    fake_ops._count[0] += 1
    return posterior_noise_ref(moments, eps, noise, channels, scaling_factor, sigma)


NAMES = ("conv3x3_down", "vae_posterior_noise")
