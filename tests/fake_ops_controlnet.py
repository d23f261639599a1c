"""TEST-ONLY stand-ins for ops.conv3x3_small and ops.controlnet_add_residuals in plain PyTorch on the CPU, used next to
tests/fake_ops.py by the ControlNet CPU wiring tests.  Never imported by the product."""
import torch
import torch.nn.functional as F


def conv3x3_small(x, w_packed, bias=None, *, stride=1, silu=False, nchw=False, out=None):
    xf = x.float() if nchw else x.float().permute(0, 3, 1, 2)
    cout, k = w_packed.shape
    w = w_packed.float().reshape(cout, 3, 3, k // 9).permute(0, 3, 1, 2)
    y = F.conv2d(xf, w, None if bias is None else bias.float(), stride=stride, padding=1)
    y = (F.silu(y) if silu else y).permute(0, 2, 3, 1).to(x.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y.contiguous()


def controlnet_add_residuals(skips, residuals, scale, skip_row0s):
    for k, (s, r, r0) in enumerate(zip(skips, residuals, skip_row0s)):
        flat = s.view(-1, s.shape[-1])
        rr = r.reshape(-1, s.shape[-1])
        flat[r0:r0 + rr.shape[0]] += (rr.float() * scale[k].float()).to(s.dtype)



def conv3x3(x, w_packed, bias=None, *, out=None, **kw):
    """fake_ops.conv3x3 that also honours out= (the conditioning embedding writes into the engine's static buffer)."""
    import fake_ops
    y = fake_ops.conv3x3(x, w_packed, bias, **kw)
    if out is not None:
        out.copy_(y)
        return out
    return y


NAMES = ("conv3x3_small", "controlnet_add_residuals", "conv3x3")
