"""The C-ABI library loads and exports every symbol include/stheno_b200.h declares
(no compute calls: there is no GPU in the CPU suite)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "stheno_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(sb_[A-Za-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from stheno_jl_b200 import lib
    so = lib.load()
    names = _declared()
    assert len(names) >= 22
    for n in names:
        assert hasattr(so, n), f"{n} declared in include/stheno_b200.h but not exported"
    assert set(lib.EXPORTS) == set(names)
    assert so.sb_abi_version() == 1


def test_no_gpu_fails_loudly():
    """Without a GPU the product path must raise, never fall back to a CPU implementation."""
    import numpy as np
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import stheno_jl_b200 as sb
    f = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
    with pytest.raises(sb.SthenoB200Error):
        sb.logpdf(f(sb.GPPPInput("f", np.arange(4.0)), 0.1), np.zeros(4))


def test_struct_layouts_match_header():
    from stheno_jl_b200 import lib
    assert ctypes.sizeof(lib.sb_array) == 24
    assert ctypes.sizeof(lib.sb_term) == 40
    assert ctypes.sizeof(lib.sb_block) == 40
    assert ctypes.sizeof(lib.sb_covspec) == 64
    assert ctypes.sizeof(lib.sb_noise) == 24
    assert ctypes.sizeof(lib.sb_timings) == 104
