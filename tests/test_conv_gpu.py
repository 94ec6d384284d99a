"""GPU parity of the wgmma implicit-GEMM convolution (through the C ABI) against a float64 PyTorch convolution of
the same op (this is a floating-point kernel, so a torch reference is the oracle; tolerance stated per test)."""
import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import dense

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 3e-5   # of max|ref|: bf16x3 products (2^-16) with fp32 accumulation


def to_hl(x, cp=None):
    """x (B,T,C,H,W) fp32 on cpu -> HL on device (test helper; the product path has its own CUDA layout kernels)."""
    B, T, C, H, W = x.shape
    cp = cp or dense.pad_to(C)
    xp = torch.zeros(B, T, H, W, cp)
    xp[..., :C] = x.permute(0, 1, 3, 4, 2)
    hi, lo = dense.split_hilo(xp.to(DEV))
    return dense.HL(hi.contiguous(), lo.contiguous(), C)


def from_hl(h, c0=0, c=None):
    c = c if c is not None else h.c
    y = h.hi.float() + h.lo.float()
    return y[..., c0:c0 + c].permute(0, 1, 4, 2, 3).cpu()


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(*shape, generator=g) * 2 - 1) * scale


def ref_conv2d(x, w, b, stride=1, dilation=1, padding=None):
    B, T, C, H, W = x.shape
    k = w.shape[-1]
    padding = padding if padding is not None else (k - 1) * dilation // 2
    y = F.conv2d(x.reshape(B * T, C, H, W).double(), w.double(), b.double(), stride=stride, padding=padding,
                 dilation=dilation)
    return y.view(B, T, *y.shape[1:])


def check(y, ref, tol=TOL):
    err = (y.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= tol * scale, (err, scale, err / scale)


@pytest.mark.parametrize("cin,cout,k,stride,dil,hw", [
    (64, 64, 1, 1, 1, (20, 24)),      # 1x1, partial tiles
    (35, 35, 3, 1, 1, (33, 17)),      # padded channels
    (64, 128, 3, 1, 12, (40, 40)),    # ASPP dilation
    (64, 128, 3, 2, 1, (36, 36)),     # stride 2
    (64, 64, 7, 2, 1, (50, 50)),      # decoder.first_conv
    (128, 256, 3, 1, 1, (25, 25)),    # two K blocks, BN=256
    (64, 128, 1, 2, 1, (20, 20)),     # resnet downsample 1x1 stride 2
    (256, 128, 1, 1, 1, (16, 16)),    # four K blocks
])
def test_conv2d_matches_fp64(cin, cout, k, stride, dil, hw):
    H, W = hw
    x = rnd(2, 2, cin, H, W, seed=1)
    w = rnd(cout, cin, k, k, seed=2, scale=(cin * k * k) ** -0.5)
    b = rnd(cout, seed=3)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV), stride=stride, dilation=dil)
    y = dense.conv(to_hl(x), pc)
    torch.cuda.synchronize()
    ref = ref_conv2d(x, w, b, stride=stride, dilation=dil)
    out = from_hl(y, 0, cout)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    check(out, ref)
    if pc.bn > cout:   # padded output channels are exactly zero (zero weights, zero bias)
        assert float((y.hi[..., cout:].float().abs() + y.lo[..., cout:].float().abs()).max()) == 0.0


@pytest.mark.parametrize("tune", [(1, 1), (2, 1), (1, 3), (2, 3), (3, 1), (3, 3)])
@pytest.mark.parametrize("cin,cout,k,dil,hw", [
    (64, 128, 3, 1, (40, 37)),        # weights streamed through the ring, partial tiles in x and y
    (128, 64, 3, 1, (24, 24)),        # two K blocks
    (64, 64, 1, 1, (50, 50)),         # resident weights
    (64, 256, 3, 2, (33, 33)),        # dilation 2, BN = 256 (two launches)
])
def test_every_tiling_matches_fp64(tune, cin, cout, k, dil, hw):
    """Every tiling the autotuner may pick -- with and without the shared dy-tap activation load, for every accepted
    n_sub value -- gives the same result."""
    if tune[1] == 3 and (k != 3 or dil != 1):
        pytest.skip("taps are not groupable")
    H, W = hw
    x = rnd(1, 3, cin, H, W, seed=31)
    w = rnd(cout, cin, k, k, seed=32, scale=(cin * k * k) ** -0.5)
    b = rnd(cout, seed=33)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV), dilation=dil)
    y = dense.conv(to_hl(x), pc, relu=True, tune=tune)
    torch.cuda.synchronize()
    check(from_hl(y, 0, cout), F.relu(ref_conv2d(x, w, b, dilation=dil)))


@pytest.mark.parametrize("tune", [(1, 1), (1, 3), (2, 3), (3, 3), (3, 7)])
@pytest.mark.parametrize("k,hw", [(7, (50, 46)), (3, (37, 41)), (5, (30, 30))])
def test_stride2_tap_groups(tune, k, hw):
    """Stride-2 kernels: the taps of one kernel column whose dy have the same parity share an activation load
    (7x7: groups of 4 and 3; 3x3: 2 and 1); decoder.first_conv / the ResNet stride-2 3x3s (decoder.py:22-30)."""
    H, W = hw
    x = rnd(2, 2, 64, H, W, seed=51)
    w = rnd(64, 64, k, k, seed=52, scale=(64 * k * k) ** -0.5)
    b = rnd(64, seed=53)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV), stride=2)
    y = dense.conv(to_hl(x), pc, relu=True, tune=tune)
    torch.cuda.synchronize()
    check(from_hl(y, 0, 64), F.relu(ref_conv2d(x, w, b, stride=2)))


@pytest.mark.parametrize("tune", [(1, 9), (2, 9), (1, 11), (2, 11), (3, 9), (3, 11), (3, 15), (2, 13)])
@pytest.mark.parametrize("cin,cout,k,hw,T", [
    (64, 64, 3, (40, 37), 2),         # resident weights
    (128, 35, 3, (24, 24), 3),        # two K blocks, padded Cout
    (64, 64, 1, (50, 50), 1),         # 1x1
])
def test_stacked_weight_operand(tune, cin, cout, k, hw, T):
    """bn = 64 layers may evaluate a product as A_hi x [W_hi; W_lo] (N = 128) + A_lo x W_hi (N = 64) -- two MMAs
    instead of three; the epilogue adds the two accumulator halves.  Same three product terms, same result."""
    if (tune[1] & 3) == 3 and k != 3:
        pytest.skip("taps are not groupable")
    H, W = hw
    x = rnd(1, T, cin, H, W, seed=61)
    w = rnd(cout, cin, k, k, seed=62, scale=(cin * k * k) ** -0.5)
    b = rnd(cout, seed=63)
    res = rnd(1, T, cout, H, W, seed=64)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    assert pc.bn == 64
    y = dense.conv(to_hl(x), pc, relu=True, residual=to_hl(res), tune=tune)
    torch.cuda.synchronize()
    check(from_hl(y, 0, cout), F.relu(ref_conv2d(x, w, b) + res.double()))


@pytest.mark.parametrize("tune", [(1, 1), (2, 3), (3, 3), (3, 11), (2, 9)])
def test_column_sums_from_the_epilogue(tune):
    """col_sums: per-image sums over pixels of the activated output (what the next block's pooling branches read),
    accumulated by the epilogue warps and reduced in a fixed order -> deterministic."""
    B, T, C, H, W = 2, 3, 64, 37, 29
    x = rnd(B, T, C, H, W, seed=71)
    w = rnd(40, C, 3, 3, seed=72, scale=0.05)
    b = rnd(40, seed=73)
    res = rnd(B, T, 40, H, W, seed=74)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    sums = torch.full((B * T, 64), float("nan"), device=DEV)
    y = dense.conv(to_hl(x), pc, relu=True, residual=to_hl(res), res_after_act=True, tune=tune, col_sums=sums)
    sums2 = torch.empty_like(sums)
    dense.conv(to_hl(x), pc, relu=True, residual=to_hl(res), res_after_act=True, tune=tune, col_sums=sums2)
    torch.cuda.synchronize()
    ref = F.relu(ref_conv2d(x, w, b)) + res.double()
    check(from_hl(y, 0, 40), ref)
    ref_sums = ref.sum(dim=(-2, -1)).view(B * T, 40)
    got = sums.cpu().double()
    assert torch.equal(sums, sums2), "not deterministic"
    assert float(got[:, 40:].abs().max()) == 0.0
    err = (got[:, :40] - ref_sums).abs().max().item()
    assert err <= 3e-5 * ref_sums.abs().max().item() + 1e-3, (err, ref_sums.abs().max().item())


@pytest.mark.parametrize("tune", [(1, 1), (2, 1), (3, 1)])
def test_two_destinations(tune):
    """Two 64-column 1x1 convolutions of the same input as one 128-column launch: columns [0,64) -> a window of a concat
    tensor with ReLU, columns [64,128) -> a second tensor without (temporal block: path 2 | projection)."""
    B, T, C, H, W = 2, 2, 64, 21, 35
    x = rnd(B, T, C, H, W, seed=81)
    wA, bA = rnd(35, C, 1, 1, seed=82, scale=0.1), rnd(35, seed=83)
    wB, bB = rnd(64, C, 1, 1, seed=84, scale=0.1), rnd(64, seed=85)
    wm = torch.zeros(128, C, 1, 1); wm[:35] = wA; wm[64:] = wB
    bm = torch.zeros(128); bm[:35] = bA; bm[64:] = bB
    ib = rnd(B * T, 128, seed=86); ib[:, 35:64] = 0
    pc = dense.pack_conv(wm.to(DEV), bm.to(DEV), bn=128)
    cat = dense.HL.zeros(B, T, H, W, 128, DEV)
    second = dense.HL.zeros(B, T, H, W, 64, DEV)
    dense.conv(to_hl(x), pc, out=cat, out_coff=80, n_store=48, relu=True, out2=second, out2_coff=0, n_store2=64,
               relu2=False, img_bias=(ib + bm).to(DEV), tune=tune)
    torch.cuda.synchronize()
    refA = F.relu(ref_conv2d(x, wA, bA) + ib[:, :35].view(B, T, 35, 1, 1).double())
    refB = ref_conv2d(x, wB, bB) + ib[:, 64:].view(B, T, 64, 1, 1).double()
    check(from_hl(cat, 80, 35), refA)
    check(from_hl(second, 0, 64), refB)
    assert float(cat.hi[..., :80].float().abs().max()) == 0.0                # nothing outside the window
    assert float((cat.hi[..., 115:].float().abs() + cat.lo[..., 115:].float().abs()).max()) == 0.0   # padded columns: zeros


def test_pair_tiling_with_fused_epilogues():
    """CTA-pair tiling with residual, per-image bias and odd image sizes (the peer CTA's rows fall off the image)."""
    B, T, C, H, W = 2, 2, 64, 9, 21
    x = rnd(B, T, C, H, W, seed=41)
    w = rnd(64, C, 3, 3, seed=42, scale=0.05)
    b = rnd(64, seed=43)
    res = rnd(B, T, 64, H, W, seed=44)
    ib = rnd(B * T, 64, seed=45)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    base = ref_conv2d(x, w, b) + ib.view(B, T, 64, 1, 1).double()
    ib = ib + b.view(1, 64)
    for tune in ((3, 1), (3, 3)):
        y = dense.conv(to_hl(x), pc, relu=True, img_bias=ib.to(DEV), residual=to_hl(res), res_after_act=True, tune=tune)
        check(from_hl(y), F.relu(base) + res.double())


@pytest.mark.parametrize("tune", [None, (1, 1), (2, 3), (3, 1), (3, 3), (3, 7), (2, 5)])
def test_causal_conv3d(tune):
    """CausalConv3d (2,3,3): time padded on the left only (temporal.py:252-273); tap groups that only see the zero
    padding in time (frame 0, dt = -1) are skipped by the kernel."""
    B, T, C, H, W = 2, 3, 35, 24, 20
    x = rnd(B, T, C, H, W, seed=4)
    w = rnd(35, C, 2, 3, 3, seed=5, scale=0.05)
    b = rnd(35, seed=6)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    y = dense.conv(to_hl(x), pc, relu=True, tune=tune)
    xp = F.pad(x.permute(0, 2, 1, 3, 4).double(), (1, 1, 1, 1, 1, 0))
    ref = F.relu(F.conv3d(xp, w.double(), b.double())).permute(0, 2, 1, 3, 4)
    check(from_hl(y, 0, 35), ref)


def test_epilogue_fusions():
    B, T, C, H, W = 1, 3, 64, 19, 21
    x = rnd(B, T, C, H, W, seed=7)
    w = rnd(64, C, 3, 3, seed=8, scale=0.05)
    b = rnd(64, seed=9)
    res = rnd(B, T, 64, H, W, seed=10)
    ib = rnd(B * T, 64, seed=11)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    base = ref_conv2d(x, w, b) + ib.view(B, T, 64, 1, 1).double()
    ib = ib + b.view(1, 64)          # the per-image table replaces the bias vector, so it carries it
    # residual before the activation (ResNet BasicBlock), written at a channel offset of a wider tensor
    out = dense.HL.zeros(B, T, H, W, 192, DEV)
    dense.conv(to_hl(x), pc, out=out, out_coff=64, relu=True, img_bias=ib.to(DEV), residual=to_hl(res))
    check(from_hl(out, 64, 64), F.relu(base + res.double()))
    assert float(out.hi[..., :64].float().abs().max()) == 0.0 and float(out.hi[..., 128:].float().abs().max()) == 0.0
    # residual after the activation (TemporalBlock skip)
    y = dense.conv(to_hl(x), pc, relu=True, img_bias=ib.to(DEV), residual=to_hl(res), res_after_act=True)
    check(from_hl(y), F.relu(base) + res.double())
    # fp32 NCHW output of the first 5 channels with sigmoid
    o32 = torch.empty(B * T, 5, H, W, device=DEV)
    dense.conv(to_hl(x), pc, img_bias=ib.to(DEV), out_f32=o32, n_valid=5, sigmoid=True)
    check(o32.view(B, T, 5, H, W).cpu(), torch.sigmoid(base[:, :, :5]), tol=1e-5)


def test_channel_window_input():
    """cin_off: read a 64-channel window of a wider (concat) tensor."""
    x = rnd(1, 1, 128, 16, 16, seed=12)
    w = rnd(64, 64, 1, 1, seed=13, scale=0.1)
    b = torch.zeros(64)
    pc = dense.pack_conv(w.to(DEV), b.to(DEV))
    y = dense.conv(to_hl(x), pc, cin_off=64)
    check(from_hl(y), ref_conv2d(x[:, :, 64:], w, b))


def test_fused_head_epilogue():
    """3x3 conv -> BN(folded) -> ReLU -> 1x1 conv(+bias) of two decoder heads evaluated in one launch (decoder.py:38-52):
    the hidden tensor is never stored; each head writes its own contiguous fp32 NCHW tensor."""
    B, T, C, H, W = 1, 2, 64, 18, 22
    x = rnd(B, T, C, H, W, seed=20)
    w3 = rnd(128, C, 3, 3, seed=21, scale=0.05)          # two heads' 3x3 kernels concatenated along N
    b3 = rnd(128, seed=22)
    w1a, b1a = rnd(2, 64, seed=23, scale=0.2), rnd(2, seed=24)
    w1b, b1b = rnd(1, 64, seed=25, scale=0.2), rnd(1, seed=26)
    pc = dense.pack_conv(w3.to(DEV), b3.to(DEV))
    w2 = torch.zeros(3, 128); w2[:2, :64] = w1a; w2[2:, 64:] = w1b
    oa = torch.empty(B * T, 2, H, W, device=DEV); ob = torch.empty(B * T, 1, H, W, device=DEV)
    dense.conv(to_hl(x), pc, relu=True, store=False,
               head={"w": w2.to(DEV).contiguous(), "b": torch.cat([b1a, b1b]).to(DEV), "outs": [(oa, 0), (oa, 1), (ob, 0)],
                     "sigmoid_mask": 0b100})
    hid = F.relu(ref_conv2d(x, w3, b3)).view(B * T, 128, H, W)
    ra = F.conv2d(hid[:, :64], w1a.double().view(2, 64, 1, 1), b1a.double())
    rb = torch.sigmoid(F.conv2d(hid[:, 64:], w1b.double().view(1, 64, 1, 1), b1b.double()))
    check(oa.cpu(), ra)
    check(ob.cpu(), rb, tol=1e-5)
