"""TEST-ONLY stand-in for ops.controlnet_add_residuals_multi in plain PyTorch on the CPU, used next to
tests/fake_ops_controlnet.py by the Multi-ControlNet CPU tests.  Never imported by the product."""


def controlnet_add_residuals_multi(skips, residuals_per_net, scales_per_net, skip_row0s):
    for k, (s, r0) in enumerate(zip(skips, skip_row0s)):
        flat = s.view(-1, s.shape[-1])
        acc = None
        for rs, sc in zip(residuals_per_net, scales_per_net):
            add = (rs[k].reshape(-1, s.shape[-1]).float() * sc[k].float()).to(s.dtype)
            acc = add if acc is None else acc + add
        flat[r0:r0 + acc.shape[0]] += acc


NAMES = ("controlnet_add_residuals_multi",)
