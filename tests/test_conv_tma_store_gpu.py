"""The convolution kernel's hi/lo outputs leave the SM as TMA stores of whole 8 x 16-pixel tiles, clipped by the output
tensor maps.  These cases check the clipping against the float64 tap-sum reference (tests/conv_reference.py): maps
whose last tiles overhang the right edge, the bottom edge or both; a channel window (out_coff > 0, n_store below the
column block) inside a wider destination whose other channels, and the memory behind the tensor, must keep their
prior contents; the second destination's window; one and several column blocks per pixel tile."""
import pytest
import torch

from stp3_b200 import dense
from tests import conv_reference as R
from tests.test_conv_gpu import DEV, TOL, rnd, to_hl

gpu = pytest.mark.gpu
SENTINEL = -1234.5          # exact in bf16
BLOCKS = {"one block": 0, "128-column blocks": 0, "64-column blocks": dense.BLOCKS64}


def packed(taps, cin, cout, seed):
    k = 3 if taps == 9 else 1
    w = rnd(cout, cin, k, k, seed=seed, scale=(cin * k * k) ** -0.5)
    return dense.pack_conv(w.to(DEV), rnd(cout, seed=seed + 1).to(DEV))


def guarded(n_img, H, W, cp, guard=4096):
    """HL destination (n_img, 1, H, W, cp) at the start of sentinel-filled buffers `guard` elements longer."""
    n = n_img * H * W * cp
    bufs = [torch.full((n + guard,), SENTINEL, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
    return dense.HL(*(b[:n].view(n_img, 1, H, W, cp) for b in bufs), cp), bufs, n


def untouched(t):
    return bool((t == SENTINEL).all())


def close(got, ref):
    err, scale = float((got.double() - ref.reshape(got.shape)).abs().max()), float(ref.abs().max())
    assert err <= TOL * scale, (err, scale)


# (H, W): the last tile row / column overhangs the bottom / right edge, or neither
MAPS = {"exact": (16, 32), "right": (16, 37), "bottom": (13, 32), "both": (21, 27), "smaller than a tile": (5, 9)}


@gpu
@pytest.mark.parametrize("hw", list(MAPS))
@pytest.mark.parametrize("taps", [1, 9])
def test_channel_window_in_a_wider_destination(hw, taps):
    """n_store = 40 of a 64-column convolution into channels [72, 112) of a 192-channel tensor: the stored window matches
    the reference, every other channel and the memory behind the tensor keep the sentinel."""
    H, W = MAPS[hw]
    n_img, coff, n_store = 3, 72, 40
    x = to_hl(rnd(n_img, 1, 64, H, W, seed=1))
    pc = packed(taps, 64, 64, 2)
    out, bufs, n = guarded(n_img, H, W, 192)
    dense.conv(x, pc, relu=True, out=out, out_coff=coff, n_store=n_store)
    ref = R.epilogue(R.tap_sum(x.hi, x.lo, pc), pc, dict(relu=True, out=out, n_store=n_store))["y"]
    close(out.hi[..., coff:coff + n_store].double() + out.lo[..., coff:coff + n_store].double(), ref)
    for t in (out.hi, out.lo):
        assert untouched(t[..., :coff]) and untouched(t[..., coff + n_store:])
    assert all(untouched(b[n:]) for b in bufs)


@gpu
@pytest.mark.parametrize("hw", list(MAPS))
@pytest.mark.parametrize("blocks", list(BLOCKS))
def test_column_blocks_on_ragged_maps(hw, blocks):
    """A 128-column convolution in one block, 256 columns in two 128-column blocks, 256 columns in four 64-column
    blocks: every block's tile boxes land in their channels and nowhere behind the tensor."""
    H, W = MAPS[hw]
    n_img = 2
    cout = 128 if blocks == "one block" else 256
    x = to_hl(rnd(n_img, 1, 64, H, W, seed=3))
    pc = packed(9, 64, cout, 4)
    out, bufs, n = guarded(n_img, H, W, cout)
    dense.conv(x, pc, relu=True, out=out, tune=(0, 3 + BLOCKS[blocks]))
    close(R.join(out), R.epilogue(R.tap_sum(x.hi, x.lo, pc), pc, dict(relu=True, out=out))["y"])
    assert all(untouched(b[n:]) for b in bufs)


@gpu
@pytest.mark.parametrize("hw", ["exact", "both"])
def test_second_destination_window(hw):
    """Two 64-column convolutions in one launch: columns [0, 48) into channels [8, 56) of a 64-channel tensor, columns
    [64, 104) into channels [16, 56) of another 128-channel tensor, each with its own activation."""
    H, W = MAPS[hw]
    n_img = 2
    x = to_hl(rnd(n_img, 1, 64, H, W, seed=5))
    pc = packed(1, 64, 128, 6)
    out, bufs, n = guarded(n_img, H, W, 64)
    out2, bufs2, n2 = guarded(n_img, H, W, 128)
    dense.conv(x, pc, relu=True, out=out, out_coff=8, n_store=48, out2=out2, out2_coff=16, n_store2=40, relu2=False)
    ref = R.epilogue(R.tap_sum(x.hi, x.lo, pc), pc, dict(relu=True, out=out, n_store=48, out2=out2, n_store2=40))
    close(out.hi[..., 8:56].double() + out.lo[..., 8:56].double(), ref["y"])
    close(out2.hi[..., 16:56].double() + out2.lo[..., 16:56].double(), ref["y2"])
    for t in (out.hi, out.lo):
        assert untouched(t[..., :8]) and untouched(t[..., 56:])
    for t in (out2.hi, out2.lo):
        assert untouched(t[..., :16]) and untouched(t[..., 56:])
    assert all(untouched(b[n:]) for b in bufs) and all(untouched(b[n2:]) for b in bufs2)
