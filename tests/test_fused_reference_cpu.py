"""The fp64 reference of the back-to-back kernels (tests/fused_reference.py), checked without a GPU:
  - against a direct F.conv2d / F.conv3d composition of the same operation on synthetic descriptors (a 1-tap branch,
    9-tap branches with unequal vertical and horizontal rates, in_cstride > cin, two K blocks, the no-ReLU tail, T = 1,
    both block chain layouts, identity and projection residual).  The module-level check, the reference run from
    DeepLabHead / TemporalBlock packed tables against the fp64 oracle, is tests/test_fused_packing_cpu.py;
  - its model mode against its exact mode: three bf16 products per stage and the hi/lo split of P stay within a few
    2^-16 of the exact result, and differ from it;
  - the argument checks of stp3_aspp_fused_fwd / stp3_block_fused_fwd, which all come before the driver is asked for
    cuTensorMapEncodeTiled, so they answer on a machine without a GPU."""
import ctypes
import os

import pytest
import torch

from stp3_b200 import _lib
from tests import fused_cases as FC
from tests import fused_reference as FR


def _x64(h):
    return h.hi.double() + h.lo.double()


@pytest.mark.parametrize("rates,cin,cs,n_out,relu", [
    ([None, (2, 3)], 64, 128, 128, True),               # 1-tap + 9-tap branch, in_cstride > cin
    ([None, (1, 5), (4, 2), (9, 30)], 64, 64, 128, True),   # four branches, the last one's taps beyond the map
    ([(1, 1)], 128, 192, 40, False),                    # the tail instance: two K blocks, no ReLU, padded rows
])
def test_aspp_reference_vs_direct_convolution(rates, cin, cs, n_out, relu):
    B, T, H, W = 2, 1, 11, 19
    case = FC.aspp_case(cin, rates, n_out=n_out, seed=3)
    x = FC.planes(B, T, H, W, cin, cs, seed=4)
    ib = FC.rnd(B * T, 128, seed=5, scale=0.3)
    got = FR.aspp(x.hi, x.lo, case.pa, ib, relu=relu)
    want = FC.aspp_direct(case, _x64(x)[..., :cin].reshape(B * T, H, W, cin).permute(0, 3, 1, 2), ib, relu=relu)
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 1e-12, err
    n64 = FR.aspp(x.hi, x.lo, case.pa, ib, relu=relu, n_store=64)
    assert torch.equal(n64, got[..., :64])


@pytest.mark.parametrize("layout,proj,T,cs,x_cs", [(0, True, 3, 64, 64), (0, False, 1, 64, 128), (1, False, 2, 64, 128),
                                                   (1, True, 1, 48, 64)])
def test_block_reference_vs_direct_convolution(layout, proj, T, cs, x_cs):
    B, H, W = 2, 9, 17
    case = FC.block_case(layout, proj, cs=cs, seed=7)
    mid = FC.planes(B, T, H, W, 128, 128, seed=8)
    x = FC.planes(B, T, H, W, cs, x_cs, seed=9)
    hid, ib = FC.rnd(B * T, 128, seed=10, scale=0.3), FC.rnd(B * T, 64, seed=11, scale=0.3)
    rb = FC.rnd(B * T, 64, seed=12, scale=0.3) if proj else None
    got, sums = FR.block_tail(mid.hi, mid.lo, x.hi, x.lo, case.pb, hid, ib, rb)
    to5 = lambda h: _x64(h).permute(0, 4, 1, 2, 3)        # noqa: E731
    want = FC.block_direct(case, to5(mid), to5(x), hid, ib, rb)
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 1e-12, err
    assert torch.allclose(sums, want.sum(dim=(1, 2)), rtol=0, atol=1e-9 * float(want.abs().sum(dim=(1, 2)).max()))


def test_model_mode_is_the_three_product_evaluation():
    case = FC.aspp_case(64, [None, (2, 2)], seed=13)
    x = FC.planes(1, 2, 10, 18, 64, 64, seed=14)
    ib = FC.rnd(2, 128, seed=15, scale=0.3)
    ex, mo = FR.aspp(x.hi, x.lo, case.pa, ib), FR.aspp(x.hi, x.lo, case.pa, ib, model=True)
    d = float((ex - mo).abs().max() / ex.abs().max())
    assert 0 < d < 1e-4, d
    bc = FC.block_case(0, True, seed=16)
    mid, xx = FC.planes(1, 2, 9, 17, 128, 128, seed=17), FC.planes(1, 2, 9, 17, 64, 64, seed=18)
    args = (mid.hi, mid.lo, xx.hi, xx.lo, bc.pb, FC.rnd(2, 128, seed=19), FC.rnd(2, 64, seed=20), FC.rnd(2, 64, seed=21))
    (ex, _), (mo, _) = FR.block_tail(*args), FR.block_tail(*args, model=True)
    d = float((ex - mo).abs().max() / ex.abs().max())
    assert 0 < d < 1e-4, d
    # P's split: hi = bf16(p), lo = bf16(p - hi) of the fp32 value
    hi, lo = FR.split(torch.tensor([1.0 + 2.0 ** -7 + 2.0 ** -12 + 2.0 ** -30], dtype=torch.float64))
    assert float(hi) == 1.0 + 2.0 ** -7 and float(lo) == 2.0 ** -12


# ----------------------------------------------------------------------------------------------- refusals
FAKE = 1 << 20   # a non-null, aligned device address: every call below is refused before it is dereferenced


def _lib_built():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


def _aspp_desc(**kw):
    d = _lib.AsppDesc()
    d.B, d.T, d.H, d.W, d.in_cstride, d.cin, d.n_br = 1, 1, 16, 32, 64, 64, 2
    d.n_taps[0], d.n_taps[1] = 1, 9
    for i in range(9):
        d.taps[1][i][0], d.taps[1][i][1] = (i // 3 - 1) * 12, (i % 3 - 1) * 12
    d.out_cstride, d.out_coff, d.no_relu, d.n_store = 128, 0, 0, 128
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_aspp_refuses_bad_descriptors_without_a_gpu():
    L = _lib_built()

    def call(d):
        return L.stp3_aspp_fused_fwd(ctypes.byref(d), FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None), L.stp3_last_error()
    no_centre = _aspp_desc()
    no_centre.taps[0][0][0] = 1
    five = _aspp_desc(n_br=5)
    for d, msg in [(no_centre, b"centre tap"), (_aspp_desc(n_store=96), b"n_store must be 64 or 128"),
                   (_aspp_desc(out_coff=8, out_cstride=256), b"16-channel aligned offset"),
                   (_aspp_desc(n_br=0), b"1 .. 4 branches"), (five, b"1 .. 4 branches")]:
        rc, err = call(d)
        assert rc == -1 and msg in err, (msg, err)
    if not torch.cuda.is_available():       # the valid descriptor passes every check and stops at the driver lookup
        rc, err = call(_aspp_desc())
        assert rc != 0 and b"cuTensorMapEncodeTiled" in err, err


def _chain(c, src, cin_off, taps, n_mma, tmem_col, k_lo, k_hi):
    c.src, c.cin_off, c.n_taps, c.n_mma, c.tmem_col, c.k_lo, c.k_hi = src, cin_off, len(taps), n_mma, tmem_col, k_lo, k_hi
    for i, t in enumerate(taps):
        c.taps[i][0], c.taps[i][1], c.taps[i][2] = t


def _block_desc(proj=True):
    """the three-path layout of block 1 (three 35-channel paths at N = 48, projection)"""
    d = _lib.BlockDesc()
    d.B, d.T, d.H, d.W, d.mid_cstride, d.x_cstride, d.out_cstride, d.n_chain = 1, 3, 16, 32, 128, 64, 64, 3
    t233 = [(it - 1, iy - 1, ix - 1) for it in range(2) for ix in range(3) for iy in range(3)]
    t133 = [(0, iy - 1, ix - 1) for ix in range(3) for iy in range(3)]
    _chain(d.chain[0], 0, 0, t233, 48, 0, 0, 48)
    _chain(d.chain[1], 0, 64, t133, 48, 48, 0, 48)
    _chain(d.chain[2], 1, 0, [(0, 0, 0)], 48, 96, 0, 64)
    d.has_res_proj = int(proj)
    _chain(d.res, 1, 0, [(0, 0, 0)], 64, 0, 0, 64)
    pc = [48 * k + 8 * q for k in range(3) for q in range(5)] + [-1]
    for i, v in enumerate(pc):
        d.piece_col[i] = v
    return d


def test_block_refuses_bad_descriptors_without_a_gpu():
    L = _lib_built()

    def call(d, res_bias=FAKE):
        rc = L.stp3_block_fused_fwd(ctypes.byref(d), FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, res_bias, FAKE, FAKE,
                                    None, None, 0, None)
        return rc, L.stp3_last_error()
    wide = _block_desc()
    _chain(wide.chain[0], 0, 0, [(0, 0, 0)], 64, 0, 0, 48)             # N = 64 in the three-path layout
    gap = _block_desc()
    gap.piece_col[15] = 112                                            # a piece after the chains' pieces
    other = _block_desc()
    _chain(other.res, 1, 0, [(0, 0, 0)], 64, 0, 0, 48)                 # the projection over other K steps than path 2
    for d, rb, msg in [(wide, FAKE, b"not a compiled chain layout"), (gap, FAKE, b"consecutive"),
                       (_block_desc(proj=False), FAKE, b"res_bias is given exactly when"),
                       (other, FAKE, b"shares the last chain's activations")]:
        rc, err = call(d, rb)
        assert rc == -1 and msg in err, (msg, err)
    if not torch.cuda.is_available():
        rc, err = call(_block_desc())
        assert rc != 0 and b"cuTensorMapEncodeTiled" in err, err
