"""CPU: the C-ABI shared library loads and exports every symbol include/stp3_b200.h declares (no compute)."""
import ctypes
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


FAKE = 1 << 20   # a non-null, aligned device address: every call below is refused before it is dereferenced


def lift_desc(**kw):
    """A valid stp3_lift_splat_desc (1 sample x 3 frames, 64 channels, 200 x 200 grid) with fields overridden by kw."""
    f = dict(cam_M=FAKE, cam_t=FAKE, ego_R=FAKE, ego_t=FAKE, xs=FAKE, ys=FAKE, ds=FAKE, bev_off=(-50.0, -50.0, -10.0),
             bev_res=(0.5, 0.5, 20.0), nx=200, ny=200, nz=1, discount=0.5, B=1, S=3, N=6, D=48, Hf=28, Wf=60, C=64,
             feat_layout=0, use_depth_distribution=1, f_begin=0, f_count=0)
    f.update(kw)
    for k in ("bev_off", "bev_res"):
        f[k] = (ctypes.c_float * 3)(*f[k])
    return _lib.LiftSplatDesc(**f)


def lift_fwd(desc, ranks_out=None, out_layout=0, n_peers=0):
    L = _lib.lib()
    peers = (ctypes.c_void_p * 1)(FAKE) if n_peers else None
    return L.stp3_lift_splat_fwd(desc, FAKE, FAKE, ranks_out, None, FAKE, 1 << 40, FAKE, out_layout, n_peers, peers, None)


def test_workspace_query_and_argument_errors_through_descriptor():
    L = _lib.lib()
    assert L.stp3_lift_splat_workspace_bytes(lift_desc()) == 3 * 64 * 200 * 200 * 4 + ((3 * 200 * 200 + 255) // 256) * 256 + 1250 * 3 * 64 * 4
    assert L.stp3_lift_splat_workspace_bytes(lift_desc(B=0)) == 0
    # frame mode: the f_count raw frames are laid out as f_count samples of one frame
    assert L.stp3_lift_splat_workspace_bytes(lift_desc(f_begin=1, f_count=2)) == 2 * 64 * 200 * 200 * 4 + ((2 * 200 * 200 + 255) // 256) * 256 + 2 * 1250 * 64 * 4
    assert L.stp3_lift_splat_bwd_scratch_bytes(lift_desc()) == 3 * 200 * 200 * 64 * 4
    # null pointers are rejected before anything touches the GPU
    desc = lift_desc(cam_M=None, cam_t=None, ego_R=None, ego_t=None, xs=None, ys=None, ds=None)
    rc = L.stp3_lift_splat_fwd(desc, None, None, None, None, None, 0, None, 0, 0, None, None)
    assert rc == -1 and b"null" in L.stp3_last_error()


def test_lift_splat_descriptor_rules():
    """One descriptor per rule, each breaking only that rule: refused with STP3_EINVAL (-1) and the rule's own message
    before any CUDA call.  Each rule reads a different field, so this also pins the ctypes mirror's layout."""
    L = _lib.lib()
    cases = {
        "receptive field S=9": lambda: lift_fwd(lift_desc(S=9)),
        "nz=2": lambda: lift_fwd(lift_desc(nz=2)),
        "frame range outside": lambda: lift_fwd(lift_desc(f_begin=2, f_count=2), out_layout=1),
        "frame mode writes no ranks_out": lambda: lift_fwd(lift_desc(f_begin=1, f_count=1), ranks_out=FAKE, out_layout=1),
        "frame mode writes fp32 channels-last": lambda: lift_fwd(lift_desc(f_begin=1, f_count=1), out_layout=0),
        "peer outputs need frame mode": lambda: lift_fwd(lift_desc(), out_layout=1, n_peers=1),
        "feat must be NCHW": lambda: L.stp3_lift_splat_bwd(lift_desc(feat_layout=1), FAKE, FAKE, FAKE, FAKE, 1 << 40, FAKE,
                                                           FAKE, None),
    }
    for msg, call in cases.items():
        assert call() == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())


def test_ops_refuse_cpu_tensors():
    import torch
    from stp3_b200 import ops
    t = torch.zeros(1, 1, 1, 2, 2, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.lift_splat(t, t, t, t, t, t, t, t, t, [0, 0, 0], [1, 1, 1], [2, 2, 1], 0.5)
