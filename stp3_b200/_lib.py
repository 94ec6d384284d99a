"""ctypes loader for libstp3_b200.so (the C ABI declared in include/stp3_b200.h).

There is NO fallback: if the library is missing or was not built, using an op raises.  The library is
built in-tree (stp3_b200/csrc/Makefile, driven by __graft_entry__.build()), so the package is importable from the
repository tree.
"""
import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstp3_b200.so")
_lib = None

# name -> (restype, argtypes); lists every symbol of include/stp3_b200.h (tests/test_abi.py checks that).
# Device pointers travel as integers (c_void_p).
_V = ctypes.c_void_p
_I = ctypes.c_int
_F = ctypes.c_float
_SZ = ctypes.c_size_t
_FP = ctypes.POINTER(ctypes.c_float)
class ConvDesc(ctypes.Structure):
    """Mirror of stp3_conv_desc (include/stp3_b200.h)."""
    _fields_ = [("B", _I), ("T", _I), ("H", _I), ("W", _I), ("T_total", _I), ("t0", _I), ("in_cstride", _I), ("cin_off", _I), ("cin", _I),
                ("Ho", _I), ("Wo", _I), ("stride", _I), ("ntaps", _I), ("taps", (ctypes.c_byte * 3) * 49),
                ("bn", _I), ("out_cstride", _I), ("out_coff", _I), ("n_store", _I), ("relu", _I), ("res_mode", _I),
                ("res_cstride", _I), ("res_coff", _I), ("n_valid", _I), ("sigmoid", _I), ("tune_n_sub", _I), ("tune_group", _I),
                ("n_cols", _I), ("col_sums", _V), ("col_sums_scratch", _V), ("col_sums_scratch_bytes", _SZ),
                ("y2_hi", _V), ("y2_lo", _V), ("out2_cstride", _I), ("out2_coff", _I), ("n_store2", _I), ("relu2", _I),
                ("k_lo", _I), ("k_hi", _I), ("f32_layout", _I)]


class AsppDesc(ctypes.Structure):
    """Mirror of stp3_aspp_desc (include/stp3_b200.h)."""
    _fields_ = [("B", _I), ("T", _I), ("H", _I), ("W", _I), ("in_cstride", _I), ("cin", _I), ("n_br", _I),
                ("n_taps", _I * 4), ("taps", ((ctypes.c_byte * 2) * 9) * 4), ("out_cstride", _I), ("out_coff", _I),
                ("no_relu", _I), ("n_store", _I)]


class BlockChain(ctypes.Structure):
    """Mirror of stp3_block_chain (include/stp3_b200.h)."""
    _fields_ = [("src", _I), ("cin_off", _I), ("n_taps", _I), ("taps", (ctypes.c_byte * 3) * 18), ("n_mma", _I),
                ("tmem_col", _I), ("k_lo", _I), ("k_hi", _I)]


class BlockDesc(ctypes.Structure):
    """Mirror of stp3_block_desc (include/stp3_b200.h)."""
    _fields_ = [("B", _I), ("T", _I), ("H", _I), ("W", _I), ("mid_cstride", _I), ("x_cstride", _I), ("out_cstride", _I),
                ("n_chain", _I), ("chain", BlockChain * 3), ("has_res_proj", _I), ("res", BlockChain), ("piece_col", _I * 16)]


class ConvHead(ctypes.Structure):
    """Mirror of stp3_conv_head (include/stp3_b200.h)."""
    _fields_ = [("n_out", _I), ("w", _V), ("b", _V), ("out", _V * 8), ("img_stride", ctypes.c_longlong * 8),
                ("sigmoid_mask", _I)]


SIGNATURES = {
    "stp3_abi_version": (_I, []),
    "stp3_conv_col_sums_scratch_bytes": (_SZ, [_I, _I]),
    "stp3_build_info": (ctypes.c_char_p, []),
    "stp3_last_error": (ctypes.c_char_p, []),
    "stp3_lift_splat_workspace_bytes": (_SZ, [_I, _I, _I, _I, _I]),
    "stp3_lift_splat_workspace_init": (_I, [_V, _SZ, _V]),
    "stp3_f32_to_hilo": (_I, [_V, _I, _I, _I, _I, _I, _I, _V, _V, _V]),
    "stp3_hilo_to_f32": (_I, [_V, _V, _I, _I, _I, _I, _I, _I, _V, _V]),
    "stp3_spatial_sum": (_I, [_V, _V, _I, _I, _I, _V, _V]),
    "stp3_pool_bias": (_I, [_V, _I, _I, _I, _I, _F, _I, _V, _I, _V, _V, _I, _V, _I, _V, _V, _I, _I, _V]),
    "stp3_small_linear": (_I, [_V, _V, _I, _I, _I, _V, _V, _I, _I, _V]),
    "stp3_upsample2x_add": (_I, [_V, _V, _I, _I, _I, _I, _V, _V, _I, _I, _V, _V, _I, _I, _I, _V]),
    "stp3_lift_splat_frames_fwd": (_I, [_V, _I, _V, _V, _V, _V, _V, _V, _V, _V, _FP, _FP, _I, _I, _I,
                                        _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _V, _SZ, _V, _V]),
    "stp3_block_fused_scratch_bytes": (_SZ, [_I]),
    "stp3_block_fused_fwd": (_I, [ctypes.POINTER(BlockDesc), _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _SZ, _V]),
    "stp3_aspp_fused_fwd": (_I, [ctypes.POINTER(AsppDesc), _V, _V, _V, _V, _V, _V, _V, _V]),
    "stp3_lift_splat_bwd_scratch_bytes": (_SZ, [_I, _I, _I, _I, _I]),
    "stp3_lift_splat_bwd": (_I, [_V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _FP, _FP, _I, _I, _I, _F,
                                 _I, _I, _I, _I, _I, _I, _I, _I, _V, _SZ, _V, _V, _V]),
    "stp3_lift_splat_frames_allgather_fwd": (_I, [_V, _I, _V, _V, _V, _V, _V, _V, _V, _V, _FP, _FP, _I, _I, _I,
                                                  _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _V, _SZ, _I,
                                                  ctypes.POINTER(ctypes.c_void_p), _V]),
    "stp3_bev_discount": (_I, [_V, _I, _I, _I, _I, _I, _F, _V, _V, _V]),
    "stp3_conv_fwd": (_I, [ctypes.POINTER(ConvDesc), _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, ctypes.POINTER(ConvHead), _V]),
    "stp3_lift_splat_fwd": (_I, [_V, _I, _V, _V, _V, _V, _V, _V, _V, _V, _FP, _FP,
                                 _I, _I, _I, _F, _I, _I, _I, _I, _I, _I, _I, _I,
                                 _V, _V, _V, _SZ, _V, _I, _V]),
}


def build(verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into stp3_b200/libstp3_b200.so (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout[-4000:])
        print(res.stderr[-4000:])
    if res.returncode != 0:
        raise RuntimeError("building libstp3_b200.so failed")
    return LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(stp3_b200 has no CPU or PyTorch fallback)")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is not exported
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def check(code: int, what: str):
    if code != 0:
        raise RuntimeError(f"{what} failed ({code}): {lib().stp3_last_error().decode()}")
