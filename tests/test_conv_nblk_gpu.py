"""Convolutions of 128 / 256 columns as (pixel tile, column block) work items of one launch (stp3_conv_desc.tune_bn):
every low-resolution decoder layer and a few awkward maps under 128-column blocks, 64-column stacked and 64-column
plain blocks against the float64 tap-sum reference (tests/conv_reference.py), the epilogue's fusions with more than one
block, bitwise agreement of a 256-column convolution with its two 128-column halves run on their own, and the
combinations the launcher refuses.  The host counts (work items, ring depths) need no GPU."""
import ctypes
import os
import sys

import pytest
import torch

from stp3_b200 import _lib, dense
from tests import conv_reference as R
from tests.test_conv_gpu import DEV, TOL, rnd, to_hl

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import conv_bench  # noqa: E402

gpu = pytest.mark.gpu
BLOCKS = {"128": 0, "64 stacked": dense.BLOCKS64 + 8, "64 plain": dense.BLOCKS64}
# (taps, cin, cout, stride, (H, W) of the input, images)
MAPS = [pytest.param(*layer[:4], (layer[4], layer[4]), 12, id=f"{layer[0]}x{layer[1]}-{layer[2]}s{layer[3]}@{layer[5]}")
        for layer in dict.fromkeys(conv_bench.LOW_RES_LAYERS) if layer[2] >= 128] + [
    pytest.param(9, 64, 256, 1, (23, 27), 12, id="ragged"),
    pytest.param(9, 128, 256, 1, (8, 16), 1, id="one tile"),
    pytest.param(9, 64, 128, 1, (13, 7), 3, id="13x7"),
]


def packed(taps, cin, cout, stride, seed):
    k = 3 if taps == 9 else 1
    w = rnd(cout, cin, k, k, seed=seed, scale=(cin * k * k) ** -0.5)
    return dense.pack_conv(w.to(DEV), rnd(cout, seed=seed + 1).to(DEV), stride=stride)


def reference(x, pc, **kw):
    return R.epilogue(R.tap_sum(x.hi, x.lo, pc), pc, kw)


def close(got, ref, tol=TOL):
    err, scale = float((got.double() - ref.reshape(got.shape)).abs().max()), float(ref.abs().max())
    assert err <= tol * scale, (err, scale)


@gpu
@pytest.mark.parametrize("blocks", list(BLOCKS))
@pytest.mark.parametrize("taps,cin,cout,stride,hw,n_img", MAPS)
def test_decoder_layers_in_column_blocks(taps, cin, cout, stride, hw, n_img, blocks):
    x = to_hl(rnd(n_img, 1, cin, *hw, seed=5))
    pc = packed(taps, cin, cout, stride, 6)
    runs = []
    for _ in range(2):
        y = dense.conv(x, pc, relu=True, tune=(0, 3 + BLOCKS[blocks]))
        runs.append((y.hi.clone(), y.lo.clone()))
    close(R.join(y), reference(x, pc, relu=True, out=True)["y"])
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), "not repeatable"


@gpu
@pytest.mark.parametrize("group", [1, 3])
def test_one_launch_of_two_blocks_equals_the_two_halves_bit_for_bit(group):
    """256 columns in 128-column blocks: the same arithmetic per element as each half run as a 128-column convolution of
    its own (how 256 columns ran before they became blocks of one launch)."""
    n_img, H, W = 12, 25, 25
    x, res = to_hl(rnd(n_img, 1, 256, H, W, seed=11)), to_hl(rnd(n_img, 1, 256, H, W, seed=12))
    pc = packed(9, 256, 256, 1, 13)
    y = dense.conv(x, pc, relu=True, residual=res, tune=(0, group))
    halves = dense.HL.zeros(n_img, 1, H, W, 256, DEV)
    for c in (0, 128):
        half = dense.PackedConv(pc.w[:, :, :, c:c + 128].contiguous(), pc.bias[c:c + 128].contiguous(), pc.taps,
                                pc.cin_p, 128, 128, 1)
        dense.conv(x, half, relu=True, residual=res, res_coff=c, out=halves, out_coff=c, tune=(0, group + 4))
    assert torch.equal(y.hi, halves.hi) and torch.equal(y.lo, halves.lo)


@gpu
def test_stacked_blocks_equal_the_stacked_64_column_kernel_bit_for_bit():
    n_img, H, W = 3, 19, 21
    x = to_hl(rnd(n_img, 1, 64, H, W, seed=21))
    pc = packed(9, 64, 128, 1, 22)
    y = dense.conv(x, pc, tune=(0, 3 + dense.BLOCKS64 + 8))
    for c in (0, 64):
        part = dense.PackedConv(pc.w[:, :, :, c:c + 64].contiguous(), pc.bias[c:c + 64].contiguous(), pc.taps,
                                pc.cin_p, 64, 64, 1)
        z = dense.conv(x, part, tune=(0, 3 + 4 + 8))
        assert torch.equal(y.hi[..., c:c + 64], z.hi) and torch.equal(y.lo[..., c:c + 64], z.lo)


@gpu
@pytest.mark.parametrize("blocks", list(BLOCKS))
@pytest.mark.parametrize("after_act", [False, True])
def test_residual_image_bias_and_a_partly_stored_last_block(blocks, after_act):
    """res_mode 1 / 2 at a channel offset of a wider residual, a per-image bias table, and n_store = 200 of 256 columns
    written into a window of a concat tensor: the last 64-column block stores 8 columns, the last 128-column one 72."""
    n_img, H, W = 5, 21, 19
    x, res = to_hl(rnd(n_img, 1, 64, H, W, seed=31)), to_hl(rnd(n_img, 1, 320, H, W, seed=32))
    pc = packed(9, 64, 256, 1, 33)
    ib = (rnd(n_img, 256, seed=34).to(DEV) + pc.bias).contiguous()
    out = dense.HL.zeros(n_img, 1, H, W, 264, DEV)
    kw = dict(relu=True, residual=res, res_coff=64, res_after_act=after_act, img_bias=ib, out=out, out_coff=56, n_store=200)
    dense.conv(x, pc, tune=(0, 3 + BLOCKS[blocks]), **kw)
    close(R.join(out)[..., 56:256], reference(x, pc, **kw)["y"])
    assert float(out.hi[..., :56].float().abs().max()) == 0.0 and float(out.hi[..., 256:].float().abs().max()) == 0.0


@gpu
@pytest.mark.parametrize("blocks", list(BLOCKS))
@pytest.mark.parametrize("nhwc", [False, True])
def test_fp32_outputs(blocks, nhwc):
    n_img, H, W, nv = 4, 17, 18, 200
    x = to_hl(rnd(n_img, 1, 128, H, W, seed=41))
    pc = packed(1, 128, 200, 1, 42)
    o = torch.zeros((n_img, H, W, nv) if nhwc else (n_img, nv, H, W), device=DEV)
    kw = dict(out_f32=o, n_valid=nv, out_f32_nhwc=nhwc, sigmoid=not nhwc)
    dense.conv(x, pc, store=False, tune=(0, 1 + BLOCKS[blocks]), **kw)
    close(o, reference(x, pc, **kw)["f32"], tol=TOL if nhwc else 1e-5)


def _desc(bn=256, **kw):
    d = _lib.ConvDesc(B=1, T=1, H=16, W=16, in_cstride=64, cin=64, Ho=16, Wo=16, stride=1, ntaps=1, bn=bn,
                      out_cstride=bn, **kw)
    return d


def test_refused_combinations():
    """A fused head, a second destination and col_sums need every column in one CTA: refused with STP3_EINVAL before
    anything touches a device, and so are block widths the kernel does not have."""
    L = _lib.lib()
    fake = 1 << 20
    info = _lib.ConvTilingInfo()
    for d in (_desc(128, tune_bn=64, y2_hi=fake, y2_lo=fake), _desc(128, tune_bn=64, col_sums=fake),
              _desc(256, tune_bn=32), _desc(64, tune_bn=128)):
        assert L.stp3_conv_tiling(ctypes.byref(d), 132, ctypes.byref(info)) == -1
        assert b"tune_bn" in L.stp3_last_error()
    head = _lib.ConvHead(n_out=1, w=fake, b=fake)
    head.out[0] = fake
    d = _desc(128, tune_bn=64)
    assert L.stp3_conv_fwd(ctypes.byref(d), fake, fake, fake, fake, None, None, None, None, None, None,
                           ctypes.byref(head), None) == -1
    assert b"tune_bn" in L.stp3_last_error()
    assert L.stp3_conv_tiling(ctypes.byref(d), 132, ctypes.byref(info)) == 0 and info.items == 4


def test_host_counts_of_the_low_resolution_layers():
    rows = {(r["layer"], r["map"]): r for r in conv_bench.count_layers(132)}
    r = rows[("9x256->256", "12x25x25")]
    assert r["128"]["items"] == 192 and r["64s"]["items"] == r["64p"]["items"] == 384
    assert r["128"]["a_stages"] == r["128"]["b_stages"] == 2
    assert min(r["64s"]["a_stages"], r["64s"]["b_stages"], r["64p"]["a_stages"], r["64p"]["b_stages"]) >= 3
    r = rows[("9x128->128", "12x50x50")]
    assert r["128"]["items"] == 336 and r["64s"]["items"] == 672 and r["64s"]["waves"] == round(672 / 132, 2)
    assert min(r["64s"]["a_stages"], r["64s"]["b_stages"]) >= 3
    assert not any(v["resident"] for r in rows.values() for k, v in r.items() if k in ("64s", "64p"))
    assert set(rows[("1x128->64", "12x50x50")]) == {"layer", "map", "128"}        # 64 columns: one block either way


def test_untuned_choice_of_blocks():
    """Without timing: 64-column stacked blocks where 128-column items make fewer than two waves of the SMs."""
    pc256 = dense.pack_conv(torch.zeros(256, 64, 1, 1), torch.zeros(256))
    pc128 = dense.pack_conv(torch.zeros(128, 64, 1, 1), torch.zeros(128))
    pc64 = dense.pack_conv(torch.zeros(64, 64, 1, 1), torch.zeros(64))
    assert dense.untuned_blocks(pc256, 96, 132) == dense.BLOCKS64 + 8      # 25 x 25: 192 items of 128 columns
    assert dense.untuned_blocks(pc128, 336, 132) == 0                      # 50 x 50: 336 items
    assert dense.untuned_blocks(pc128, 96, 132) == dense.BLOCKS64 + 8
    assert dense.untuned_blocks(pc64, 96, 132) == 0
