"""CPU: the C-ABI shared library loads and exports every symbol include/stp3_b200.h declares (no compute)."""
import os
import re

import pytest

from stp3_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "stp3_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(stp3_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    syms = header_symbols()
    assert syms, "no symbols parsed from the header"
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/stp3_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in stp3_b200/_lib.py"
    assert L.stp3_abi_version() >= 1
    assert b"sm_90a" in L.stp3_build_info()


def test_workspace_query_and_argument_errors():
    L = _lib.lib()
    assert L.stp3_lift_splat_workspace_bytes(1, 3, 64, 200, 200) == 3 * 64 * 200 * 200 * 4 + ((3 * 200 * 200 + 255) // 256) * 256 + 1250 * 3 * 64 * 4
    assert L.stp3_lift_splat_workspace_bytes(0, 3, 64, 200, 200) == 0
    # null pointers are rejected before anything touches the GPU
    import ctypes
    z3 = (ctypes.c_float * 3)(0, 0, 0)
    rc = L.stp3_lift_splat_fwd(None, 0, None, None, None, None, None, None, None, None, z3, z3, 200, 200, 1, 0.5,
                               1, 1, 1, 1, 1, 1, 1, 1, None, None, None, 0, None, 0, None)
    assert rc == -1 and b"null" in L.stp3_last_error()


def test_ops_refuse_cpu_tensors():
    import torch
    from stp3_b200 import ops
    t = torch.zeros(1, 1, 1, 2, 2, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.lift_splat(t, t, t, t, t, t, t, t, t, [0, 0, 0], [1, 1, 1], [2, 2, 1], 0.5)
