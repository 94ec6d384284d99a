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
_LL = ctypes.c_longlong
_ULL = ctypes.c_ulonglong


class LiftSplatDesc(ctypes.Structure):
    """Mirror of stp3_lift_splat_desc (include/stp3_b200.h)."""
    _fields_ = [("cam_M", _V), ("cam_t", _V), ("ego_R", _V), ("ego_t", _V), ("xs", _V), ("ys", _V), ("ds", _V),
                ("bev_off", _F * 3), ("bev_res", _F * 3), ("nx", _I), ("ny", _I), ("nz", _I), ("discount", _F),
                ("B", _I), ("S", _I), ("N", _I), ("D", _I), ("Hf", _I), ("Wf", _I), ("C", _I),
                ("feat_layout", _I), ("use_depth_distribution", _I), ("f_begin", _I), ("f_count", _I)]


_LSD = ctypes.POINTER(LiftSplatDesc)


class LiftSplatPlan(ctypes.Structure):
    """Mirror of stp3_lift_splat_kernel_plan (include/stp3_b200.h)."""
    _fields_ = [("tma_rules", _I), ("scatter", _I), ("scatter_tw", _I), ("finalize", _I), ("finalize_vec", _I),
                ("finalize_smax", _I), ("finalize_lpp", _I), ("channel_groups", _I)]


class ConvDesc(ctypes.Structure):
    """Mirror of stp3_conv_desc (include/stp3_b200.h)."""
    _fields_ = [("B", _I), ("T", _I), ("H", _I), ("W", _I), ("T_total", _I), ("t0", _I), ("in_cstride", _I), ("cin_off", _I), ("cin", _I),
                ("Ho", _I), ("Wo", _I), ("stride", _I), ("ntaps", _I), ("taps", (ctypes.c_byte * 3) * 49),
                ("bn", _I), ("out_cstride", _I), ("out_coff", _I), ("n_store", _I), ("relu", _I), ("res_mode", _I),
                ("res_cstride", _I), ("res_coff", _I), ("n_valid", _I), ("sigmoid", _I), ("tune_n_sub", _I), ("tune_group", _I),
                ("n_cols", _I), ("col_sums", _V), ("col_sums_scratch", _V), ("col_sums_scratch_bytes", _SZ),
                ("y2_hi", _V), ("y2_lo", _V), ("out2_cstride", _I), ("out2_coff", _I), ("n_store2", _I), ("relu2", _I),
                ("k_lo", _I), ("k_hi", _I), ("f32_layout", _I), ("swish", _I), ("w_img_stride", _LL), ("tune_bn", _I)]


class ConvTilingInfo(ctypes.Structure):
    """Mirror of stp3_conv_tiling_info (include/stp3_b200.h)."""
    _fields_ = [("bn_blk", _I), ("stacked", _I), ("tiles", _I), ("items", _I), ("ctas", _I), ("a_stages", _I),
                ("b_stages", _I), ("resident", _I)]


class DwDesc(ctypes.Structure):
    """Mirror of stp3_dw_desc (include/stp3_b200.h)."""
    _fields_ = [("n_img", _I), ("H", _I), ("W", _I), ("Ho", _I), ("Wo", _I), ("k", _I), ("stride", _I), ("pad_t", _I),
                ("pad_l", _I), ("C", _I), ("in_cstride", _I), ("out_cstride", _I)]


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


class HlSlot(ctypes.Structure):
    """Mirror of stp3_hl_slot (include/stp3_b200.h)."""
    _fields_ = [("hi", _V), ("lo", _V), ("cstride", _I), ("coff", _I), ("t_total", _I), ("t0", _I)]


_HS = ctypes.POINTER(HlSlot)


class PlanDesc(ctypes.Structure):
    """Mirror of stp3_plan_desc (include/stp3_b200.h)."""
    _fields_ = [("B", _I), ("N", _I), ("T", _I), ("H", _I), ("W", _I), ("dx", _F * 2), ("bx", _F * 2),
                ("fp0", _I * 4), ("fp1", _I * 4), ("safety", _F), ("headway", _F), ("lrdivider", _F), ("comfort", _F),
                ("progress", _F), ("volume", _F), ("rule", _F), ("safety_w", _F * 2), ("headway_dist", _F), ("lane_dist", _F),
                ("n_hd", _I), ("traj_c", _I), ("G", _I)]


_PD = ctypes.POINTER(PlanDesc)

SIGNATURES = {
    "stp3_abi_version": (_I, []),
    "stp3_conv_col_sums_scratch_bytes": (_SZ, [_I, _I]),
    "stp3_conv_tiling": (_I, [ctypes.POINTER(ConvDesc), _I, ctypes.POINTER(ConvTilingInfo)]),
    "stp3_build_info": (ctypes.c_char_p, []),
    "stp3_last_error": (ctypes.c_char_p, []),
    "stp3_lift_splat_workspace_bytes": (_SZ, [_LSD]),
    "stp3_lift_splat_workspace_init": (_I, [_V, _SZ, _V]),
    "stp3_f32_to_hilo": (_I, [_V, _I, _I, _I, _I, _I, _I, _V, _V, _V]),
    "stp3_f32_to_plane": (_I, [_V, _I, _I, _I, _I, _I, _I, _I, _V, _V]),
    "stp3_hilo_to_f32": (_I, [_V, _V, _I, _I, _I, _I, _I, _I, _V, _V]),
    "stp3_spatial_sum": (_I, [_V, _V, _I, _I, _I, _V, _V]),
    "stp3_pool_bias": (_I, [_V, _I, _I, _I, _I, _F, _I, _V, _I, _V, _V, _I, _V, _I, _V, _V, _I, _I, _V]),
    "stp3_small_linear": (_I, [_V, _V, _I, _I, _I, _V, _V, _I, _I, _V]),
    "stp3_upsample2x_add": (_I, [_V, _V, _I, _I, _I, _I, _V, _V, _I, _I, _V, _V, _I, _I, _I, _V]),
    "stp3_block_fused_scratch_bytes": (_SZ, [_I]),
    "stp3_block_fused_fwd": (_I, [ctypes.POINTER(BlockDesc), _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _SZ, _V]),
    "stp3_aspp_fused_fwd": (_I, [ctypes.POINTER(AsppDesc), _V, _V, _V, _V, _V, _V, _V, _V]),
    "stp3_lift_splat_bwd_scratch_bytes": (_SZ, [_LSD]),
    "stp3_lift_splat_bwd": (_I, [_LSD, _V, _V, _V, _V, _SZ, _V, _V, _V]),
    "stp3_lift_splat_bwd_cl": (_I, [_LSD, _V, _V, _V, _V, _SZ, _V, _V, _V]),
    "stp3_bev_discount": (_I, [_V, _I, _I, _I, _I, _I, _F, _V, _V, _V]),
    "stp3_conv_fwd": (_I, [ctypes.POINTER(ConvDesc), _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, ctypes.POINTER(ConvHead), _V]),
    "stp3_conv_fwd_plane": (_I, [ctypes.POINTER(ConvDesc), _I, _V, _V, _V, _V, _V, _V]),
    "stp3_conv_tiling_op": (_I, [ctypes.POINTER(ConvDesc), _I, _I, ctypes.POINTER(ConvTilingInfo)]),
    "stp3_lift_splat_fwd": (_I, [_LSD, _V, _V, _V, _V, _V, _SZ, _V, _I, _I, ctypes.POINTER(_V), _V]),
    "stp3_lift_splat_plan": (_I, [_LSD, _V, _V, _I, _I, ctypes.POINTER(LiftSplatPlan)]),
    # deterministic mode (torch.use_deterministic_algorithms)
    "stp3_lift_splat_det_workspace_bytes": (_SZ, [_LSD]),
    "stp3_lift_splat_fwd_det": (_I, [_LSD, _V, _V, _V, _V, _V, _SZ, _V, _I, _I, ctypes.POINTER(_V), _V]),
    "stp3_spatial_sum_det_scratch_bytes": (_SZ, [_I, _I, _I]),
    "stp3_spatial_sum_det": (_I, [_V, _V, _I, _I, _I, _V, _V, _SZ, _V]),
    # train mode of the decoder and the DeepLab head
    "stp3_conv_wgrad_scratch_bytes": (_SZ, [_I, _I, _I, _I, _I, _I, _I, _I]),
    "stp3_conv_wgrad": (_I, [_V, _I, _I, _I, _I, _I, _V, _I, _I, _I, _I, _I, _I, _I, _I, _I, _V, _SZ, _V, _V]),
    "stp3_bn_scratch_bytes": (_SZ, [_LL, _I]),
    "stp3_bn_stats": (_I, [_V, _LL, _I, _I, _F, _F, _V, _V, _V, _V, _V, _V, _SZ, _V]),
    "stp3_bn_apply": (_I, [_V, _LL, _I, _I, _V, _V, _V, _V, _V, _I, _I, _F, _ULL, _ULL, _V, _I, _V, _V, _I, _V]),
    "stp3_bn_apply_plane": (_I, [_V, _LL, _I, _I, _V, _V, _V, _V, _V, _I, _I, _F, _ULL, _ULL, _V, _I, _V, _I, _I, _V]),
    "stp3_image_channel_sums_scratch_bytes": (_SZ, [_I, _LL, _I]),
    "stp3_image_channel_sums": (_I, [_V, _I, _LL, _I, _I, _V, _V, _SZ, _V]),
    "stp3_bn_bwd_reduce": (_I, [_V, _I, _V, _I, _V, _I, _V, _V, _LL, _I, _V, _V, _V, _SZ, _V]),
    "stp3_bn_bwd_apply": (_I, [_V, _I, _V, _I, _V, _I, _V, _V, _V, _V, _V, _LL, _I, _V, _I, _V, _I, _V]),
    "stp3_bn_local_moments": (_I, [_V, _LL, _I, _I, _V, _V, _SZ, _V]),
    "stp3_bn_merge_finalize": (_I, [_V, _I, _I, _F, _F, _V, _V, _V, _V, _V, _V]),
    "stp3_bn_bwd_local_sums": (_I, [_V, _I, _V, _I, _V, _I, _V, _V, _LL, _I, _V, _V, _SZ, _V]),
    "stp3_bn_bwd_merge_sums": (_I, [_V, _I, _I, _V, _V, _V]),
    "stp3_bn_bwd_apply_global": (_I, [_V, _I, _V, _I, _V, _I, _V, _V, _V, _V, _V, _LL, _LL, _I, _V, _I, _V, _I, _V]),
    "stp3_upsample2x_f32": (_I, [_V, _I, _I, _I, _I, _V, _V]),
    "stp3_upsample2x_bwd": (_I, [_V, _I, _I, _I, _I, _V, _V]),
    "stp3_upsample2x_window_f32": (_I, [_V, _I, _I, _I, _I, _V, _I, _I, _V]),
    "stp3_upsample2x_window_bwd": (_I, [_V, _I, _I, _I, _I, _I, _I, _V, _V]),
    "stp3_phase_interleave": (_I, [_V, _V, _V, _V, _I, _I, _I, _I, _V, _V]),
    "stp3_sigmoid_bwd": (_I, [_V, _V, _LL, _V, _V]),
    # train mode of the TemporalBlocks
    "stp3_conv3d_wgrad_scratch_bytes": (_SZ, [_I, _I, _I, _I, _I, _I, _I, _I, _I]),
    "stp3_conv3d_wgrad": (_I, [_V, _I, _I, _I, _I, _I, _I, _V, _I, _I, _I, _I, _I, _V, _SZ, _V, _V]),
    # one-plane (autocast) train mode: operand STP3_OPERAND_BF16 / STP3_OPERAND_F16
    "stp3_conv_wgrad_plane": (_I, [_I, _V, _I, _I, _I, _I, _I, _V, _I, _I, _I, _I, _I, _I, _I, _I, _I, _V, _SZ, _V, _V]),
    "stp3_conv3d_wgrad_plane": (_I, [_I, _V, _I, _I, _I, _I, _I, _I, _V, _I, _I, _I, _I, _I, _V, _SZ, _V, _V]),
    "stp3_temporal_pair_mean": (_I, [_V, _I, _I, _I, _I, _V, _V]),
    # EfficientNet trunk
    "stp3_effnet_stem": (_I, [_V, _I, _I, _I, _I, _I, _I, _I, _V, _V, _I, _I, _V, _V, _V]),
    "stp3_dw_sums_scratch_bytes": (_SZ, [ctypes.POINTER(DwDesc)]),
    "stp3_dw_fwd": (_I, [ctypes.POINTER(DwDesc), _V, _V, _V, _V, _V, _V, _V, _V, _SZ, _V]),
    "stp3_se_proj_weight_elems": (_LL, [_I, _I]),
    "stp3_se_gate": (_I, [_V, _I, _I, _I, _F, _V, _V, _I, _V, _V, _V, _I, _V, _V, _V]),
    # train mode of the EfficientNet trunk
    "stp3_effnet_stem_raw": (_I, [_V, _I, _I, _I, _I, _I, _I, _I, _V, _I, _V, _V]),
    "stp3_effnet_stem_wgrad_scratch_bytes": (_SZ, [_I, _I, _I, _I]),
    "stp3_effnet_stem_wgrad": (_I, [_V, _I, _I, _I, _I, _I, _I, _I, _V, _I, _V, _V, _SZ, _V]),
    "stp3_dw_fwd_raw": (_I, [ctypes.POINTER(DwDesc), _V, _V, _V, _V]),
    "stp3_dw_dgrad": (_I, [ctypes.POINTER(DwDesc), _V, _V, _V, _V]),
    "stp3_dw_wgrad_scratch_bytes": (_SZ, [ctypes.POINTER(DwDesc)]),
    "stp3_dw_wgrad": (_I, [ctypes.POINTER(DwDesc), _V, _V, _V, _V, _SZ, _V]),
    "stp3_trunk_bn_act": (_I, [_V, _LL, _I, _LL, _V, _V, _V, _V, _I, _V, _V, _V, _V, _V, _V, _I, _V]),
    "stp3_trunk_bn_act_bwd": (_I, [_V, _V, _LL, _I, _LL, _V, _V, _V, _V, _I, _V, _V, _V, _V, _V]),
    "stp3_image_channel_dot_scratch_bytes": (_SZ, [_I, _LL, _I]),
    "stp3_image_channel_dot": (_I, [_V, _V, _I, _LL, _I, _V, _V, _SZ, _V]),
    "stp3_se_bwd": (_I, [_V, _V, _V, _I, _I, _F, _V, _V, _I, _V, _V, _V, _V, _V, _V]),
    # eval-mode prediction stage
    "stp3_gru_gates": (_I, [_HS, _HS, _HS, _I, _I, _LL, _I, _V]),
    "stp3_gru_update": (_I, [_HS, _HS, _HS, _HS, _HS, _I, _I, _LL, _I, _V]),
    "stp3_channel_norm_act": (_I, [_HS, _V, _V, _F, _I, _HS, _I, _HS, _I, _I, _LL, _I, _V]),
    "stp3_dw_ln": (_I, [_HS, _V, _V, _I, _V, _V, _F, _HS, _I, _I, _I, _I, _I, _V]),
    "stp3_trust_mix": (_I, [_HS, _V, _HS, _HS, _HS, _I, _I, _I, _LL, _I, _V]),
    "stp3_maxpool2_pad": (_I, [_HS, _HS, _I, _I, _I, _I, _I, _V]),
    "stp3_hl_copy": (_I, [_HS, _HS, _I, _I, _LL, _I, _V]),
    "stp3_hl_broadcast": (_I, [_V, _I, _HS, _I, _I, _LL, _I, _V]),
    # eval-mode planning
    "stp3_plan_maps": (_I, [_PD, _V, _V, _V, _V, _V, _V]),
    "stp3_plan_cost": (_I, [_PD, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V]),
    "stp3_plan_refine": (_I, [_PD, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V]),
}


# operand kinds of the train-mode convolutions (STP3_OPERAND_* of include/stp3_b200.h)
OPERAND_HILO, OPERAND_BF16, OPERAND_F16 = 0, 1, 2


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
