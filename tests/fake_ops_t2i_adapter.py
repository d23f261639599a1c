"""TEST-ONLY stand-ins for the ops the T2I-Adapter adds to the text-to-image loop (the folded pool + in_conv on
conv3x3_down, the feature injection and the MultiAdapter sum), in plain PyTorch on the CPU, used next to
tests/fake_ops.py by the T2I-Adapter CPU tests.  Never imported by the product."""
from fake_ops_controlnet import controlnet_add_residuals  # noqa: F401
from fake_ops_img2img import conv3x3_down  # noqa: F401
from fake_ops_multi_controlnet import controlnet_add_residuals_multi  # noqa: F401

NAMES = ("conv3x3_down", "controlnet_add_residuals", "controlnet_add_residuals_multi")
