"""TEST-ONLY stand-in for ops.im2col3x3_nchw_cat in plain PyTorch on the CPU, used next to tests/fake_ops.py by the
9-channel inpainting CPU wiring tests.  Never imported by the product."""
import torch

import fake_ops


def im2col3x3_nchw_cat(x0, x1, kpad, out=None):
    return fake_ops.im2col3x3_nchw(torch.cat([x0, x1.to(x0.dtype)], dim=1), kpad)


NAMES = ("im2col3x3_nchw_cat",)
