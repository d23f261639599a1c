"""TEST-ONLY stand-ins for the `relu=True` forms of imagharmony_b200.ops.linear / conv3x3 (IH_EPI_RELU: ReLU after
the residual), on top of tests/fake_ops.py, for the tiny-autoencoder CPU wiring tests.  Never imported by the product."""
import torch

import fake_ops


def linear(x, w, bias=None, *, relu=False, **kw):
    y = fake_ops.linear(x, w, bias, **kw)
    return torch.relu(y) if relu else y


def conv3x3(x, w_packed, bias=None, *, relu=False, **kw):
    y = fake_ops.conv3x3(x, w_packed, bias, **kw)
    return torch.relu(y) if relu else y


NAMES = ("linear", "conv3x3")
