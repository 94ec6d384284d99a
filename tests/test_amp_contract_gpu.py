"""GPU: the one-plane (autocast) train-mode kernels launch by launch against an fp64 model of their contract.

The model rounds every operand to fp16 / bf16 exactly as the kernels do (round to nearest even, overflow to +-inf:
torch's own fp32 -> fp16 / bf16 conversion), sums the products in fp64, and bounds each element by a few fp32 ulps of
the sum of the absolute values of its terms (the kernels accumulate in fp32).  Covered: stp3_conv_fwd_plane on the tap
sets of dense_train (3x3, dilated 3x3, 7x7 stride 2 and the stride-2 input-gradient phases, causal (2,3,3) 3-D),
stp3_conv_wgrad_plane (2-D, dilated, stride 2) and stp3_conv3d_wgrad_plane, stp3_f32_to_plane and stp3_bn_apply_plane
with dropout; inf from overflow, NaN propagation, and bitwise-repeatable weight gradients."""
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_dense as TD
from stp3_b200 import _lib, dense
from stp3_b200 import dense_train as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ULP = 2.0 ** -23
MODES = [torch.float16, torch.bfloat16]
# elementwise bar in fp32 ulps of the summed magnitudes: K-step chains of fp32 accumulation (up to 2304 terms here)
CONV_ULPS, WGRAD_ULPS = 64, 64


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rnd(t, mode):
    """what the kernels multiply: t rounded to the 16-bit type, as fp64"""
    return t.to(mode).double()


def ulp_ratio(got, ref, mag, k):
    got, ref, mag = got.double().cpu(), ref.double().cpu(), mag.double().cpu()
    return float(((got - ref).abs() / (k * ULP * mag + 1e-300)).max())


def cl(t):          # NCHW -> NHWC fp32 on the device
    return t.float().permute(0, 2, 3, 1).contiguous().to(DEV)


# ------------------------------------------------------------------------------------------------ conversions
@pytest.mark.parametrize("mode", MODES)
def test_f32_to_plane_rounds_like_torch_and_keeps_inf_nan(mode):
    x = gauss((3, 5, 7, 70), 1) * 300.0
    x[0, 0, 0, :4] = torch.tensor([1e6, -1e6, float("nan"), float("inf")])
    x[1, 1, 1, :2] = torch.tensor([65519.0, 65520.0])               # the fp16 rounding edge to inf
    x = x.to(DEV)
    p = T.to_hl(x, mode=mode)
    assert p.lo is None and p.hi.dtype == mode and p.hi.shape[-1] == 128
    got = p.hi.view(3, 5, 7, 128)
    want = x.to(mode)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got[..., :70]), nan)
    assert torch.equal(got[..., :70][~nan].view(torch.int16), want[~nan].view(torch.int16))
    assert bool((got[..., 70:] == 0).all()) and not bool(torch.signbit(got[..., 70:].float()).any())
    if mode == torch.float16:
        assert torch.isinf(got[0, 0, 0, :2]).all() and got[1, 1, 1, 0].item() == 65504.0 and torch.isinf(got[1, 1, 1, 1])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("C,p", [(64, 0.0), (64, 0.5), (35, 0.5)])
def test_bn_apply_plane_matches_bn_apply_and_its_dropout(mode, C, p):
    """y and the dropout bits equal stp3_bn_apply's (vector path C = 64, scalar path C = 35); the plane is y rounded."""
    x = gauss((2, 9, 11, C), 2).to(DEV)
    st = T.bn_stats(x, 1e-5, 0.1)
    gam, bet = gauss((C,), 3).to(DEV), gauss((C,), 4).to(DEV)
    y_ref, hl = T.bn_apply(x, st, gam, bet, relu=True, dropout=(p, 123, 7))
    y, pl = T.bn_apply(x, st, gam, bet, relu=True, dropout=(p, 123, 7), mode=mode)
    assert torch.equal(y, y_ref)
    assert pl.lo is None and pl.hi.dtype == mode
    got = pl.hi.view(2, 9, 11, -1)
    assert torch.equal(got[..., :C].view(torch.int16), y.to(mode).view(torch.int16))
    assert bool((got[..., C:] == 0).all())


def test_bn_apply_plane_overflow_is_inf():
    C = 64
    x = gauss((1, 4, 4, C), 5).to(DEV)
    st = T.bn_stats(x, 1e-5, 0.1)
    gam = torch.full((C,), 1e6, device=DEV)
    bet = torch.zeros(C, device=DEV)
    _, pl = T.bn_apply(x, st, gam, bet, relu=False, mode=torch.float16)
    assert bool(torch.isinf(pl.hi[..., :C]).any())
    # bf16 has fp32's exponent range: a finite fp32 y beyond bf16's largest value rounds to inf
    _, pl = T.bn_apply(x, st, torch.ones(C, device=DEV), torch.full((C,), 3.4e38, device=DEV), relu=False,
                       mode=torch.bfloat16)
    assert bool(torch.isinf(pl.hi[..., :C]).any())


# ------------------------------------------------------------------------------------------------ convolution fwd
CONV_GEOMS = [  # (cin, cout, k, stride, dilation, H, W)
    (64, 64, 3, 1, 1, 25, 25), (64, 128, 3, 1, 1, 50, 50), (128, 256, 3, 1, 1, 13, 17), (64, 64, 7, 2, 1, 48, 64),
    (64, 128, 3, 2, 1, 25, 25), (256, 128, 1, 1, 1, 50, 50), (64, 8, 1, 1, 1, 20, 20), (128, 64, 3, 1, 6, 20, 30),
    (35, 35, 3, 1, 1, 16, 24), (160, 64, 3, 1, 12, 14, 30)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geom", CONV_GEOMS)
def test_conv_fwd_plane_matches_rounded_fp64(mode, geom):
    cin, cout, k, stride, dil, H, W = geom
    pad = (k - 1) * dil // 2
    x = gauss((2, cin, H, W), 6)
    w = gauss((cout, cin, k, k), 7) * 0.05
    xr, wr = rnd(x, mode), rnd(w, mode)
    ref = F.conv2d(xr, wr, stride=stride, padding=pad, dilation=dil)
    mag = F.conv2d(xr.abs(), wr.abs(), stride=stride, padding=pad, dilation=dil)
    got = T.conv_raw(T.to_hl(cl(x), mode=mode), w.to(DEV), stride, dilation=dil)
    r = ulp_ratio(got.permute(0, 3, 1, 2), ref, mag, CONV_ULPS)
    print(f"{geom} {mode}: {r * CONV_ULPS:.1f} ulps of the magnitude sum")
    assert r <= 1, r


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geom", [(64, 64, 3, 1, 1), (64, 128, 3, 2, 1), (64, 64, 7, 2, 1), (128, 64, 3, 1, 6),
                                  (64, 3, 1, 1, 1), (35, 35, 3, 1, 1)])
def test_conv_dgrad_plane_matches_rounded_fp64(mode, geom):
    """input gradients: transposed / mirrored taps, dilated, and the four stride-2 phases"""
    cin, cout, k, stride, dil = geom
    H, W, pad = 25, 31, (k - 1) * dil // 2
    w = gauss((cout, cin, k, k), 8) * 0.05
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = gauss((2, cout, Ho, Wo), 9)
    gr, wr = rnd(g, mode), rnd(w, mode)
    ref = torch.nn.grad.conv2d_input((2, cin, H, W), wr, gr, stride=stride, padding=pad, dilation=dil)
    mag = torch.nn.grad.conv2d_input((2, cin, H, W), wr.abs(), gr.abs(), stride=stride, padding=pad, dilation=dil)
    got = T.conv_dgrad(cl(g), w.to(DEV), stride, H, W, dilation=dil, mode=mode)
    r = ulp_ratio(got.permute(0, 3, 1, 2), ref, mag, CONV_ULPS)
    assert r <= 1, r


def causal3d(x, w):
    """x (B, C, T, H, W), w (co, ci, kt, k, k): the TemporalBlock's causal 'same' convolution"""
    kt, k = w.shape[2], w.shape[3]
    return F.conv3d(F.pad(x, (k // 2, k // 2, k // 2, k // 2, kt - 1, 0)), w)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c,kt", [(35, 2), (64, 2), (32, 1)])
def test_conv3d_fwd_dgrad_wgrad_plane(mode, c, kt):
    B, Tn, H, W = 2, 3, 16, 24
    x = gauss((B, c, Tn, H, W), 10)
    w = gauss((c, c, kt, 3, 3), 11) * 0.05
    g = gauss((B, c, Tn, H, W), 12)
    xr, wr, gr = rnd(x, mode), rnd(w, mode), rnd(g, mode)
    # forward
    ref, mag = causal3d(xr, wr), causal3d(xr.abs(), wr.abs())
    x_cl = x.float().permute(0, 2, 3, 4, 1).reshape(B * Tn, H, W, c).contiguous().to(DEV)
    xp = T.to_hl(x_cl, mode=mode)
    xp = dense.HL(xp.hi.view(B, Tn, H, W, -1), None, c)
    got = T.conv_raw(xp, w.to(DEV), 1).view(B, Tn, H, W, c).permute(0, 4, 1, 2, 3)
    assert ulp_ratio(got, ref, mag, CONV_ULPS) <= 1
    # input gradient: the anti-causal taps
    xd = xr.clone().requires_grad_(True)
    (dx_ref,) = torch.autograd.grad(causal3d(xd, wr), xd, gr)
    xa = xr.abs().clone().requires_grad_(True)
    (dx_mag,) = torch.autograd.grad(causal3d(xa, wr.abs()), xa, gr.abs())
    g_cl = g.float().permute(0, 2, 3, 4, 1).reshape(B * Tn, H, W, c).contiguous().to(DEV)
    dx = T.conv_dgrad(g_cl, w.to(DEV), 1, H, W, T=Tn, mode=mode).view(B, Tn, H, W, c).permute(0, 4, 1, 2, 3)
    assert ulp_ratio(dx, dx_ref, dx_mag, CONV_ULPS) <= 1
    # weight gradient
    wd = wr.clone().requires_grad_(True)
    (dw_ref,) = torch.autograd.grad(causal3d(xr, wd), wd, gr)
    wa = wr.abs().clone().requires_grad_(True)
    (dw_mag,) = torch.autograd.grad(causal3d(xr.abs(), wa), wa, gr.abs())
    dw = T.conv_wgrad(x_cl.view(B, Tn, H, W, c), g_cl.view(B, Tn, H, W, c), 3, 3, 1, kt=kt, mode=mode)
    r = ulp_ratio(dw, dw_ref, dw_mag, WGRAD_ULPS)
    print(f"3-D wgrad {c} kt={kt} {mode}: {r * WGRAD_ULPS:.1f} ulps")
    assert r <= 1, r
    dw2 = T.conv_wgrad(x_cl.view(B, Tn, H, W, c), g_cl.view(B, Tn, H, W, c), 3, 3, 1, kt=kt, mode=mode)
    assert torch.equal(dw, dw2)


# ------------------------------------------------------------------------------------------------ weight gradient
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geom", [(64, 64, 3, 1, 1, 50, 50), (64, 128, 3, 2, 1, 25, 25), (64, 64, 7, 2, 1, 48, 64),
                                  (128, 128, 3, 1, 12, 20, 30), (256, 128, 1, 1, 1, 50, 50), (64, 1, 1, 1, 1, 25, 25),
                                  (35, 70, 3, 1, 1, 16, 24), (160, 64, 1, 1, 1, 14, 30)])
def test_conv_wgrad_plane_matches_rounded_fp64(mode, geom):
    cin, cout, k, stride, dil, H, W = geom
    pad = (k - 1) * dil // 2
    x = gauss((2, cin, H, W), 13)
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = gauss((2, cout, Ho, Wo), 14)
    xr, gr = rnd(x, mode), rnd(g, mode)
    shape = (cout, cin, k, k)
    ref = torch.nn.grad.conv2d_weight(xr, shape, gr, stride=stride, padding=pad, dilation=dil)
    mag = torch.nn.grad.conv2d_weight(xr.abs(), shape, gr.abs(), stride=stride, padding=pad, dilation=dil)
    dw = T.conv_wgrad(cl(x), cl(g), k, k, stride, dilation=dil, mode=mode)
    r = ulp_ratio(dw, ref, mag, WGRAD_ULPS)
    print(f"wgrad {geom} {mode}: {r * WGRAD_ULPS:.1f} ulps of the magnitude sum")
    assert r <= 1, r
    assert torch.equal(dw, T.conv_wgrad(cl(x), cl(g), k, k, stride, dilation=dil, mode=mode))


# ------------------------------------------------------------------------------------------------ inf and NaN
@pytest.mark.parametrize("mode", MODES)
def test_overflow_gives_inf_and_nan_propagates(mode):
    big = 1e6 if mode == torch.float16 else 3.4e38     # finite in fp32, beyond the 16-bit type's largest value
    x = gauss((1, 64, 12, 12), 15)
    g = gauss((1, 64, 12, 12), 16)
    w = gauss((64, 64, 3, 3), 17).to(DEV) * 0.05
    g_big = g.clone()
    g_big[0, 3, 5, 5] = big
    dw = T.conv_wgrad(cl(x), cl(g_big), 3, 3, 1, mode=mode)
    assert not bool(torch.isfinite(dw[3]).all()) and bool(torch.isfinite(dw[:3]).all())
    dx = T.conv_dgrad(cl(g_big), w, 1, 12, 12, mode=mode)
    assert not bool(torch.isfinite(dx[0, 4:7, 4:7]).all()) and bool(torch.isfinite(dx[0, 9:, 9:]).all())
    x_nan = x.clone()
    x_nan[0, 7, 4, 4] = float("nan")
    y = T.conv_raw(T.to_hl(cl(x_nan), mode=mode), w, 1)
    assert bool(torch.isnan(y[0, 3:6, 3:6]).all()) and bool(torch.isfinite(y[0, 8:, 8:]).all())
    dw = T.conv_wgrad(cl(x_nan), cl(g), 3, 3, 1, mode=mode)
    assert bool(torch.isnan(dw[:, 7]).any()) and bool(torch.isfinite(dw[:, :7]).all())


def test_one_plane_weights_need_one_plane_input():
    x = gauss((1, 8, 8, 64), 18).to(DEV)
    pc = dense.pack_conv(gauss((64, 64, 3, 3), 19).to(DEV), torch.zeros(64, device=DEV), plane=torch.float16)
    out = torch.empty((1, 8, 8, 64), device=DEV)
    with pytest.raises(AssertionError):
        dense.conv(T.to_hl(x), pc, out_f32=out, n_valid=64, out_f32_nhwc=True, store=False, tune=(0, 0))
    with pytest.raises(AssertionError):
        dense.conv(T.to_hl(x, mode=torch.bfloat16), pc, out_f32=out, n_valid=64, out_f32_nhwc=True, store=False,
                   tune=(0, 0))
    assert _lib.OPERAND_F16 == dense.PLANE_OPERAND[torch.float16]
