"""The C-ABI shared library loads on a CPU-only box and exports every symbol include/ih_api.h declares."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "ih_api.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(ih_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from imagharmony_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in ih_api.h but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature in _lib.SIGNATURES"
    assert set(_lib.SIGNATURES) == set(declared)
    assert lib.ih_version() == 2


def test_product_path_fails_loudly_without_gpu_tensors():
    import torch
    from imagharmony_b200 import ops
    from imagharmony_b200._lib import IHError
    with pytest.raises(IHError):
        ops.linear(torch.zeros(8, 8, dtype=torch.float16), torch.zeros(8, 8, dtype=torch.float16))


def test_argument_validation_returns_error_codes():
    from imagharmony_b200 import _lib
    lib = _lib.load()
    rc = lib.ih_gemm_f16(None, 0, None, None, None, 0, 0, None, 0, None, 0, 1, 1, 1, 0, 0, None)
    assert rc < 0 and b"null" in lib.ih_last_error()
    rc = lib.ih_layernorm_f16(1, 1, 1, 1, 4, 7, 1e-5, None)   # C not a multiple of 8 (checked before any launch)
    assert rc < 0


@pytest.mark.parametrize("C0,C1,B,HW,groups", [
    (1280, 0, 1, 64, 1280),    # one row lane per block: 2*groups partial sums would overrun the statistics buffer
    (2048, 0, 1, 64, 2048),
    (1280, 1280, 2, 64, 2560),
    (1280, 0, 1, 64, 0),       # no group count (and no division by zero on the host)
    (1280, 0, 1, 64, 3),       # groups does not divide C
    (4104, 0, 1, 64, 8),       # C above 4096 (the statistics buffer and 48 KiB of shared memory)
    (4096, 8, 1, 64, 32),
    (8192, 0, 1, 64, 32),
    (320, 0, 0, 64, 32),       # empty batch
    (320, 0, 1025, 64, 32),    # more images than ticket slots
    (320, 0, 2, 0, 32),        # no pixels
    (324, 0, 1, 64, 4),        # C0 not a multiple of 8
])
def test_groupnorm_rejects_unsupported_configurations(C0, C1, B, HW, groups):
    """Checked on the host before anything is launched (fake non-null pointers never reach a kernel)."""
    from imagharmony_b200 import _lib
    lib = _lib.load()
    rc = lib.ih_groupnorm_f16(1, C0, 1 if C1 else None, C1, 1, 1, 1, 1, B, HW, groups, 1e-5, 0, None)
    assert rc < 0 and b"ih_groupnorm_f16" in lib.ih_last_error(), (rc, lib.ih_last_error())
