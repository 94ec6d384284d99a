"""CPU: the float64 tap-sum reference of stp3_conv_fwd (tests/conv_reference.py), which the GPU contract tests hold the
kernel to, against PyTorch's own convolutions.  Inputs and weights sit on a 2^-15 grid in (-1, 1): at most 16
significant bits, so their bf16 hi/lo split is exact and the 'exact' tap sum must equal the fp64 convolution to
round-off."""
import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import dense, dense_train
from tests import conv_reference as R

TOL = 1e-12


def grid16(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.round((torch.rand(*shape, generator=g) * 2 - 1) * 2 ** 15) / 2 ** 15


def planes(x_cl: torch.Tensor, cp: int):
    """(B, T, H, W, C) fp32 -> hi/lo planes (B, T, H, W, cp), padding channels zero."""
    xp = torch.zeros(*x_cl.shape[:-1], cp)
    xp[..., :x_cl.shape[-1]] = x_cl
    hi, lo = dense.split_hilo(xp)
    assert torch.equal(hi.double() + lo.double(), xp.double())
    return hi, lo


def rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("cin,cout,k,stride,dil,hw,prune", [
    (64, 64, 3, 1, 1, (13, 11), False),
    (35, 40, 3, 1, 2, (9, 14), False),        # padded channels, dilation
    (64, 128, 3, 2, 1, (13, 10), False),      # stride 2, odd and even sizes
    (64, 64, 7, 2, 1, (15, 12), False),       # decoder.first_conv
    (64, 32, 1, 2, 1, (9, 9), False),
    (64, 64, 3, 1, 12, (7, 9), True),         # ASPP dilation: taps beyond the image pruned by pack_conv
])
def test_tap_sum_matches_conv2d(cin, cout, k, stride, dil, hw, prune):
    H, W = hw
    x = grid16(2, cin, H, W, seed=1)
    w = grid16(cout, cin, k, k, seed=2)
    b = grid16(cout, seed=3)
    pc = dense.pack_conv(w, b, stride=stride, dilation=dil, prune_extent=hw if prune else None)
    if prune:
        assert len(pc.taps) == 1
    hi, lo = planes(x.permute(0, 2, 3, 1).unsqueeze(1), pc.cin_p)
    got = R.tap_sum(hi, lo, pc)
    ref = F.conv2d(x.double(), w.double(), stride=stride, padding=(k - 1) * dil // 2, dilation=dil).permute(0, 2, 3, 1)
    assert got[..., :cout].shape == ref.shape
    assert rel(got[..., :cout], ref) < TOL
    assert float(got[..., cout:].abs().max() if pc.bn > cout else 0.0) == 0.0
    # the three-product model drops only lo . lo (< 2^-16 of a product)
    model = R.tap_sum(hi, lo, pc, model=True)
    assert rel(model[..., :cout], ref) < 1e-5


def test_tap_sum_matches_causal_conv3d_and_frame_windows():
    B, T, C, H, W = 2, 4, 35, 9, 12
    x = grid16(B, C, T, H, W, seed=4)
    w = grid16(40, C, 2, 3, 3, seed=5)
    pc = dense.pack_conv(w, torch.zeros(40))
    hi, lo = planes(x.permute(0, 2, 3, 4, 1), pc.cin_p)
    ref = F.conv3d(F.pad(x.double(), (1, 1, 1, 1, 1, 0)), w.double()).permute(0, 2, 3, 4, 1)   # (B, T, H, W, 40)
    got = R.tap_sum(hi, lo, pc).view(B, T, H, W, -1)
    assert rel(got[..., :40], ref) < TOL
    # frames (t0, T): frames [2, 4) of every sample; the causal tap of frame 2 reads frame 1
    got = R.tap_sum(hi, lo, pc, frames=(2, 2)).view(B, 2, H, W, -1)
    assert rel(got[..., :40], ref[:, 2:]) < TOL


def test_tap_sum_in_layout_and_channel_window():
    """in_layout: the logical input channels live at physical offsets of a concat tensor; cin_off selects a 64-channel
    aligned window of a wider tensor."""
    B, H, W = 1, 10, 7
    xa, xb = grid16(B, 20, H, W, seed=6), grid16(B, 13, H, W, seed=7)
    w = grid16(24, 33, 3, 3, seed=8)
    pc = dense.pack_conv(w, torch.zeros(24), in_layout=[(0, 20, 8), (20, 13, 40)], cin_p=64)
    assert (pc.k_lo, pc.k_hi) == (0, 64)
    phys = torch.zeros(B, 192, H, W)
    phys[:, 64 + 8:64 + 28] = xa
    phys[:, 64 + 40:64 + 53] = xb
    hi, lo = planes(phys.permute(0, 2, 3, 1).unsqueeze(1), 192)
    got = R.tap_sum(hi, lo, pc, cin_off=64)
    ref = F.conv2d(torch.cat([xa, xb], 1).double(), w.double(), padding=1).permute(0, 2, 3, 1)
    assert rel(got[..., :24], ref) < TOL
    # a layout that starts inside the first K block trims the K range at the front (k_lo > 0)
    pc2 = dense.pack_conv(w[:, :20], torch.zeros(24), in_layout=[(0, 20, 40)], cin_p=64)
    assert (pc2.k_lo, pc2.k_hi) == (32, 64)
    assert float(R.tap_sum(hi, lo, pc2, cin_off=0).abs().max()) == 0.0     # channels 40..60 of window 0 are zero
    got3 = R.tap_sum(hi, lo, pc2, cin_off=64)
    ref3 = F.conv2d(xb.double(), w[:, :13].double(), padding=1).permute(0, 2, 3, 1)
    assert rel(got3[..., :24], ref3) < TOL


@pytest.mark.parametrize("k,stride,hw", [(3, 1, (9, 8)), (3, 2, (9, 8)), (3, 2, (8, 9)), (7, 2, (11, 10)),
                                         (1, 2, (7, 6))])
def test_dgrad_phase_packs_match_conv2d_input(k, stride, hw):
    """The input gradient as stride-1 convolutions of the output gradient (dense_train.pack_dgrad), one per phase of a
    stride-2 convolution, joined by a phase interleave: equals torch.nn.grad.conv2d_input."""
    H, W = hw
    cin, cout, pad = 40, 64, (k - 1) // 2
    w = grid16(cout, cin, k, k, seed=9)
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = grid16(2, cout, Ho, Wo, seed=10)
    ref = torch.nn.grad.conv2d_input((2, cin, H, W), w.double(), g.double(), stride=stride, padding=pad)
    hi, lo = planes(g.permute(0, 2, 3, 1).unsqueeze(1), dense.pad_to(cout))
    out = torch.zeros(2, H, W, cin, dtype=torch.float64)
    for (py, px), pc in dense_train.pack_dgrad(w, stride, pad):
        if pc is None:
            continue
        Hp, Wp = (H - py + 1) // 2 if stride == 2 else H, (W - px + 1) // 2 if stride == 2 else W
        ph = R.tap_sum(hi, lo, pc, out_hw=(Hp, Wp))[..., :cin]
        if stride == 1:
            out = ph
        else:
            out[:, py::2, px::2] = ph
    assert rel(out, ref.permute(0, 2, 3, 1)) < TOL


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,cout,k,stride,dil,hw", [(64, 64, 3, 1, 1, (13, 11)), (35, 40, 3, 1, 2, (9, 14)),
                                                      (64, 128, 3, 2, 1, (13, 10)), (64, 64, 7, 2, 1, (15, 12)),
                                                      (130, 8, 1, 1, 1, (5, 6))])
def test_plane_tap_sum_matches_conv2d_of_rounded_operands(mode, cin, cout, k, stride, dil, hw):
    """one-plane weights and input: the tap sum is the fp64 convolution of the operands rounded to the plane type, and
    `absolute` is that of their magnitudes"""
    H, W = hw
    x = torch.randn(2, cin, H, W, generator=torch.Generator().manual_seed(11)) * 3
    w = torch.randn(cout, cin, k, k, generator=torch.Generator().manual_seed(12)) * 0.1
    pc = dense.pack_conv(w, torch.zeros(cout), stride=stride, dilation=dil, plane=mode)
    assert pc.w.dtype == mode and pc.w.shape == (len(pc.taps), pc.cin_p // 64, pc.bn, 64)
    xp = torch.zeros(2, 1, H, W, pc.cin_p, dtype=mode)
    xp[..., :cin] = x.permute(0, 2, 3, 1).unsqueeze(1).to(mode)
    xr, wr = x.to(mode).double(), w.to(mode).double()
    kw = dict(stride=stride, padding=(k - 1) * dil // 2, dilation=dil)
    ref = F.conv2d(xr, wr, **kw).permute(0, 2, 3, 1)
    mag = F.conv2d(xr.abs(), wr.abs(), **kw).permute(0, 2, 3, 1)
    got = R.tap_sum(xp, None, pc)
    assert rel(got[..., :cout], ref) < TOL
    assert float(got[..., cout:].abs().max() if pc.bn > cout else 0.0) == 0.0
    assert torch.equal(R.tap_sum(xp, None, pc, model=True), got)
    assert rel(R.tap_sum(xp, None, pc, absolute=True)[..., :cout], mag) < TOL
    with pytest.raises(AssertionError):
        R.tap_sum(xp, xp, pc)


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
def test_plane_tap_sum_matches_causal_conv3d_and_dgrad_phases(mode):
    """the TemporalBlocks' causal (2, 3, 3) forward over a frame window, and the stride-2 input-gradient phases, as
    one-plane tap sums"""
    B, T, C, H, W = 2, 3, 35, 9, 12
    x = torch.randn(B, C, T, H, W, generator=torch.Generator().manual_seed(13))
    w = torch.randn(40, C, 2, 3, 3, generator=torch.Generator().manual_seed(14)) * 0.1
    pc = dense.pack_conv(w, torch.zeros(40), plane=mode)
    xp = torch.zeros(B, T, H, W, pc.cin_p, dtype=mode)
    xp[..., :C] = x.permute(0, 2, 3, 4, 1).to(mode)
    ref = F.conv3d(F.pad(x.to(mode).double(), (1, 1, 1, 1, 1, 0)), w.to(mode).double()).permute(0, 2, 3, 4, 1)
    assert rel(R.tap_sum(xp, None, pc).view(B, T, H, W, -1)[..., :40], ref) < TOL
    assert rel(R.tap_sum(xp, None, pc, frames=(1, 2)).view(B, 2, H, W, -1)[..., :40], ref[:, 1:]) < TOL
    # input gradient of a 3x3 stride-2 convolution, phase by phase
    Hi, Wi, cin, cout = 9, 8, 40, 64
    wg = torch.randn(cout, cin, 3, 3, generator=torch.Generator().manual_seed(15)) * 0.1
    g = torch.randn(2, cout, 5, 4, generator=torch.Generator().manual_seed(16))
    ref = torch.nn.grad.conv2d_input((2, cin, Hi, Wi), wg.to(mode).double(), g.to(mode).double(), stride=2, padding=1)
    gp = g.permute(0, 2, 3, 1).unsqueeze(1).to(mode).contiguous()
    out = torch.zeros(2, Hi, Wi, cin, dtype=torch.float64)
    for (py, px), ph in dense_train.pack_dgrad(wg, 2, 1, plane=mode):
        Hp, Wp = (Hi - py + 1) // 2, (Wi - px + 1) // 2
        out[:, py::2, px::2] = R.tap_sum(gp, None, ph, out_hw=(Hp, Wp))[..., :cin]
    assert rel(out, ref.permute(0, 2, 3, 1)) < TOL
