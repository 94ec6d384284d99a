"""CPU: stp3_conv_tiling_op, the operand-aware tiling query the convolution contract suite counts its instantiations
with (tests/conv_reference.py tiling).  Host arithmetic only: the library loads without a GPU and no descriptor is
launched."""
import ctypes
import os

import pytest
import torch

from stp3_b200 import _lib, dense
from tests import conv_reference as R

PLANES = {"bf16": (torch.bfloat16, _lib.OPERAND_BF16), "fp16": (torch.float16, _lib.OPERAND_F16)}


@pytest.fixture(scope="module", autouse=True)
def library():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


def _w(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * 0.1


def layers():
    """(name, packed hi/lo conv, the same weights packed as one plane, geometry (B, T_total, T, H, W, Ho, Wo))"""
    out = []
    for i, (cout, cin, k, stride, dil, HW) in enumerate([
            (64, 64, 3, 1, 1, (25, 25)), (64, 128, 3, 1, 1, (50, 50)), (40, 35, 3, 1, 1, (19, 21)),
            (128, 64, 3, 1, 1, (50, 50)), (256, 128, 3, 1, 1, (13, 17)), (100, 64, 1, 1, 1, (20, 30)),
            (64, 64, 7, 2, 1, (48, 64)), (128, 160, 3, 1, 12, (14, 30)), (8, 64, 1, 1, 1, (20, 20)),
            (64, 256, 3, 1, 1, (25, 25)), (128, 128, 3, 2, 1, (25, 25))]):
        w, b = _w(cout, cin, k, k, seed=i), torch.zeros(cout)
        hl = dense.pack_conv(w, b, stride=stride, dilation=dil)
        planes = {nm: dense.pack_conv(w, b, stride=stride, dilation=dil, plane=dt) for nm, (dt, _) in PLANES.items()}
        H, W = HW
        geom = (2, 1, 1, H, W, (H + stride - 1) // stride, (W + stride - 1) // stride)
        out.append((f"{cout}x{cin}x{k}x{k} s{stride} d{dil}", hl, planes, geom))
    w = _w(64, 64, 2, 3, 3, seed=99)
    hl = dense.pack_conv(w, torch.zeros(64))
    planes = {nm: dense.pack_conv(w, torch.zeros(64), plane=dt) for nm, (dt, _) in PLANES.items()}
    out.append(("causal (2,3,3)", hl, planes, (2, 3, 3, 16, 24, 16, 24)))
    return out


def cfgs(pc):
    return [(0, 0)] + dense.tune_candidates(pc)


def test_hilo_operand_answers_as_conv_tiling():
    L = _lib.lib()
    n = 0
    for name, pc, _, geom in layers():
        for cfg in cfgs(pc):
            B, Tt, T, H, W, Ho, Wo = geom
            got = R.tiling(pc, geom, cfg, in_cstride=pc.cin_p)
            d = _lib.ConvDesc()
            d.B, d.T, d.H, d.W, d.T_total, d.in_cstride, d.cin = B, T, H, W, Tt, pc.cin_p, pc.cin_p
            d.Ho, d.Wo, d.stride, d.ntaps, d.bn, d.n_cols = Ho, Wo, pc.stride, len(pc.taps), pc.bn, pc.cout
            for i, tap in enumerate(pc.taps):
                for j in range(3):
                    d.taps[i][j] = tap[j]
            d.k_lo, d.k_hi = pc.k_lo, pc.k_hi
            d.tune_group, d.tune_bn = cfg[1] & ~dense.BLOCKS64, 64 if cfg[1] & dense.BLOCKS64 else 0
            info = _lib.ConvTilingInfo()
            assert L.stp3_conv_tiling(ctypes.byref(d), 132, ctypes.byref(info)) == 0, L.stp3_last_error()
            want = {k: getattr(info, k) for k, _ in _lib.ConvTilingInfo._fields_}
            assert {k: got[k] for k in want} == want, (name, cfg)
            n += 1
    assert n > 40


@pytest.mark.parametrize("plane", list(PLANES))
def test_plane_tilings(plane):
    """a plane never stacks; +16 runs 64-column blocks for every operand; the stacked bit changes nothing for a plane"""
    op = PLANES[plane][1]
    for name, pc, planes, geom in layers():
        pp = planes[plane]
        for cfg in cfgs(pc):
            t = R.tiling(pp, geom, cfg, in_cstride=pp.cin_p, operand=op)
            assert not t["stacked"], (name, cfg)
            if cfg[1] & dense.BLOCKS64:
                assert t["bn_blk"] == 64 and R.tiling(pc, geom, cfg, in_cstride=pc.cin_p)["bn_blk"] == 64, (name, cfg)
            if cfg[1] & 8:
                assert t == R.tiling(pp, geom, (cfg[0], cfg[1] & ~8), in_cstride=pp.cin_p, operand=op), (name, cfg)


def test_one_plane_can_keep_weights_resident_where_hilo_streams():
    """one-plane stages are half as wide, so a layer's weights can stay resident as a plane but not as a hi/lo pair"""
    found = []
    for name, pc, planes, geom in layers():
        for cfg in cfgs(pc):
            hl = R.tiling(pc, geom, cfg, in_cstride=pc.cin_p)
            for nm, (_, op) in PLANES.items():
                t = R.tiling(planes[nm], geom, cfg, in_cstride=pc.cin_p, operand=op)
                assert (t["tiles"], t["items"], t["bn_blk"]) == (hl["tiles"], hl["items"], hl["bn_blk"]), (name, cfg)
                if t["resident"] and not hl["resident"]:
                    found.append((name, cfg, nm))
    assert found
    assert any(name.startswith("64x128x3x3") for name, _, _ in found), found


def test_operand_out_of_range_is_refused():
    _, pc, _, geom = layers()[0]
    with pytest.raises(RuntimeError, match="operand"):
        R.tiling(pc, geom, (0, 0), in_cstride=64, operand=3)
