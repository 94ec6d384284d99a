"""CPU: the float64 reference of the train-mode entry points (tests/train_reference.py) against PyTorch's own
definitions of the same operations, the Philox code against the Random123 known-answer vectors, the K-split mirror
against the library's scratch sizes, and the argument refusals of the train entry points (they return before any CUDA
call, so they run without a device)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import _lib
from tests import train_reference as R


def _rand(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).float()


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    assert float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-300), float((a - b).abs().max())


# ------------------------------------------------------------------------------------------------ weight gradient
@pytest.mark.parametrize("H,W,cin,cout,k,stride,dil", [(9, 7, 5, 3, 3, 1, 1), (9, 7, 5, 3, 3, 2, 1), (8, 10, 4, 6, 7, 2, 1),
                                                       (6, 11, 3, 2, 3, 1, 4), (5, 13, 2, 3, 3, 1, 6), (1, 9, 3, 2, 3, 1, 1),
                                                       (7, 1, 3, 2, 1, 2, 1)])
def test_wgrad_matches_conv2d_weight(H, W, cin, cout, k, stride, dil):
    pad = (k - 1) * dil // 2
    x = _rand(2, H, W, cin, seed=1)
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = _rand(2, Ho, Wo, cout, seed=2)
    ref = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (cout, cin, k, k), g.double().permute(0, 3, 1, 2),
                                      stride=stride, padding=pad, dilation=dil)
    # 'same' output size: conv2d gives floor((H + 2 pad - d (k - 1) - 1) / s) + 1 = ceil(H / s) for these pads
    _close(R.wgrad(x, g, k, k, stride, pad, dil)[:, :, 0], ref)


@pytest.mark.parametrize("B,T,kt,k", [(2, 3, 2, 3), (1, 1, 2, 3), (2, 2, 3, 1), (3, 1, 1, 3)])
def test_wgrad_3d_matches_causal_conv3d_autograd(B, T, kt, k):
    H, W, cin, cout = 5, 6, 3, 4
    x = _rand(B, T, H, W, cin, seed=3)
    g = _rand(B, T, H, W, cout, seed=4)
    w = torch.zeros(cout, cin, kt, k, k, dtype=torch.float64, requires_grad=True)
    xin = F.pad(x.double().permute(0, 4, 1, 2, 3), (0, 0, 0, 0, kt - 1, 0))          # causal: kt - 1 frames on the left
    y = F.conv3d(xin, w, padding=(0, k // 2, k // 2))
    (y * g.double().permute(0, 4, 1, 2, 3)).sum().backward()
    got = R.wgrad(x.reshape(B * T, H, W, cin), g.reshape(B * T, H, W, cout), k, k, 1, k // 2, 1, kt=kt, T=T)
    _close(got, w.grad)
    if kt > T:                                  # time taps that read padding for every frame are exact zeros
        assert not got[:, :, :kt - T].any()


def test_wgrad_model_is_three_bf16_products():
    x, g = _rand(1, 6, 5, 7, seed=5), _rand(1, 6, 5, 3, seed=6)
    exact, model = R.wgrad(x, g, 3, 3, 1, 1), R.wgrad(x, g, 3, 3, 1, 1, model=True)
    e = float((exact - model).abs().max() / exact.abs().max())
    assert 0 < e < 2.0 ** -14, e              # only the lo x lo products (<= 2^-16 relative) and split roundings remain
    xh, xl = R.dense.split_hilo(x)
    gh, gl = R.dense.split_hilo(g)
    by_hand = sum(R.wgrad(a.float(), b.float(), 3, 3, 1, 1) for b, a in ((gh, xh), (gh, xl), (gl, xh)))
    _close(model, by_hand, 1e-15)


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,W,cin,cout,k,stride,dil", [(9, 7, 5, 3, 3, 1, 1), (8, 10, 4, 6, 7, 2, 1), (9, 8, 3, 4, 3, 2, 1),
                                                       (6, 11, 3, 2, 3, 1, 4)])
def test_plane_wgrad_matches_conv2d_weight_of_rounded_operands(mode, H, W, cin, cout, k, stride, dil):
    """2-D, stride 2 (odd and even) and dilated: the plane weight gradient is torch.nn.grad.conv2d_weight of x and g
    rounded to the plane type, whether they arrive as fp32 or as planes"""
    pad = (k - 1) * dil // 2
    x = _rand(2, H, W, cin, seed=21) * 3
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = _rand(2, Ho, Wo, cout, seed=22)
    ref = torch.nn.grad.conv2d_weight(x.to(mode).double().permute(0, 3, 1, 2), (cout, cin, k, k),
                                      g.to(mode).double().permute(0, 3, 1, 2), stride=stride, padding=pad, dilation=dil)
    got = R.wgrad(x, g, k, k, stride, pad, dil, plane=mode)
    _close(got[:, :, 0], ref)
    assert torch.equal(R.wgrad(x.to(mode), g.to(mode), k, k, stride, pad, dil, plane=mode), got)
    assert not torch.equal(got, R.wgrad(x, g, k, k, stride, pad, dil))       # the rounding is there


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,T,kt,k", [(2, 3, 2, 3), (1, 1, 2, 3), (2, 2, 3, 1)])
def test_plane_wgrad_3d_matches_causal_conv3d_autograd(mode, B, T, kt, k):
    H, W, cin, cout = 5, 6, 3, 4
    x = _rand(B, T, H, W, cin, seed=23)
    g = _rand(B, T, H, W, cout, seed=24)
    w = torch.zeros(cout, cin, kt, k, k, dtype=torch.float64, requires_grad=True)
    xin = F.pad(x.to(mode).double().permute(0, 4, 1, 2, 3), (0, 0, 0, 0, kt - 1, 0))
    (F.conv3d(xin, w, padding=(0, k // 2, k // 2)) * g.to(mode).double().permute(0, 4, 1, 2, 3)).sum().backward()
    got = R.wgrad(x.reshape(B * T, H, W, cin), g.reshape(B * T, H, W, cout), k, k, 1, k // 2, 1, kt=kt, T=T, plane=mode)
    _close(got, w.grad)


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
def test_bn_apply_plane_is_the_rounded_fp32_output(mode):
    """the plane reference is torch's rounding of the fp32 bn_apply output (overflow to inf, -0.0 kept) with +0
    padding channels"""
    x = _rand(50, 7, seed=25) * 4
    mean, invstd, gamma, beta = _rand(7, seed=26), _rand(7, seed=27).abs() + 0.5, _rand(7, seed=28), _rand(7, seed=29)
    y = R.bn_apply(x, mean, invstd, gamma, beta)["y"].float()
    y[0, 0], y[1, 1] = -0.0, 1e6
    pl = R.bn_apply_plane(y, 16, mode)
    assert pl.dtype == mode and pl.shape == (50, 16)
    assert torch.equal(pl[:, :7].view(torch.int16), y.to(mode).view(torch.int16))
    assert not pl[:, 7:].view(torch.int16).any() and torch.signbit(pl[0, 0].float())
    assert torch.isinf(pl[1, 1].float()) == (mode == torch.float16)


def test_wgrad_split_plan():
    assert R.wgrad_split(240000, 18, 35, 35) == (30, 8000)            # causal (2,3,3) 35 -> 35, B = 2, T = 3, 200x200
    assert R.wgrad_split(2 * 48 * 64, 9, 64, 64) == (24, 256)
    n, per = R.wgrad_split(2 * 130 * 130, 1, 128, 128)                # rounding per up to 64 leaves empty splits
    assert -(-2 * 130 * 130 // per) < n
    assert R.wgrad_split(100, 1, 8, 8) == (1, 128)


# ------------------------------------------------------------------------------------------------ BatchNorm
@pytest.mark.parametrize("relu,res", [(False, False), (True, True)])
def test_batchnorm_matches_batchnorm2d_autograd(relu, res):
    N, C, H, W = 3, 5, 4, 6
    bn = torch.nn.BatchNorm2d(C, eps=2.0 ** -10, momentum=0.25).double().train()
    with torch.no_grad():
        bn.weight.copy_(torch.linspace(0.5, 1.5, C)), bn.bias.copy_(torch.linspace(-0.2, 0.3, C))
        bn.running_mean.copy_(torch.linspace(0, 1, C)), bn.running_var.copy_(torch.linspace(1, 2, C))
    x = (_rand(N, C, H, W, seed=7) * 3 + 1).double().requires_grad_(True)
    r = _rand(N, C, H, W, seed=8).double() if res else None
    G = _rand(N, C, H, W, seed=9).double()
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    y = bn(x) + (r if res else 0)
    y = y.relu() if relu else y
    (y * G).sum().backward()
    cl = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C)        # noqa: E731
    st = R.bn_stats(cl(x.detach()), bn.eps, bn.momentum, rm0, rv0)
    _close(st["run_mean"], bn.running_mean), _close(st["run_var"], bn.running_var)
    ap = R.bn_apply(cl(x.detach()), st["mean"], st["invstd"], bn.weight, bn.bias, cl(r) if res else None, relu)
    _close(ap["y"], cl(y.detach()))
    ymask = ap["y"] if relu else None
    red = R.bn_bwd_reduce(cl(G), ymask, cl(x.detach()), st["mean"], st["invstd"])
    _close(red["sum_g"], bn.bias.grad), _close(red["sum_gx"], bn.weight.grad)
    bw = R.bn_bwd_apply(cl(G), ymask, cl(x.detach()), st["mean"], st["invstd"], bn.weight, red["sum_g"], red["sum_gx"])
    _close(bw["dx"], cl(x.grad))
    _close(bw["g_masked"], cl(G) * (cl(y.detach()) > 0) if relu else cl(G))


def test_image_channel_sums_and_pair_mean():
    x = _rand(3, 20, 6, seed=10)
    _close(R.image_channel_sums(x)["sums"], x.double().sum(1))
    m = _rand(2, 4, 3, seed=11).double().requires_grad_(True)
    # AvgPool3d((2, 1, 1)) with time padding 1, count_include_pad=False, on m as (B, C, T, 1, 1)
    pooled = F.avg_pool3d(m.permute(0, 2, 1)[..., None, None], (2, 1, 1), stride=1, padding=(1, 0, 0),
                          count_include_pad=False)[..., 0, 0].permute(0, 2, 1)
    _close(R.temporal_pair_mean(m.detach())["out"], pooled.detach())
    G = _rand(2, 5, 3, seed=12).double()
    (pooled * G).sum().backward()
    _close(R.temporal_pair_mean(G, adjoint=True)["out"], m.grad)


# ------------------------------------------------------------------------------------------------ elementwise
@pytest.mark.parametrize("h,w", [(5, 7), (1, 4), (3, 1), (1, 1)])
def test_upsample_pair_matches_interpolate_autograd(h, w):
    x = _rand(2, 3, h, w, seed=13).double().requires_grad_(True)
    y = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    G = _rand(2, 3, 2 * h, 2 * w, seed=14).double()
    (y * G).sum().backward()
    _close(R.upsample2x(x.detach().permute(0, 2, 3, 1))["y"], y.detach().permute(0, 2, 3, 1))
    _close(R.upsample2x_bwd(G.permute(0, 2, 3, 1))["gx"], x.grad.permute(0, 2, 3, 1))


def test_phase_interleave_and_sigmoid_bwd():
    H, W = 5, 4
    full = _rand(2, H, W, 3, seed=15)
    phases = [full[:, py::2, px::2].contiguous() for py in range(2) for px in range(2)]
    assert torch.equal(R.phase_interleave(phases, H, W), full)
    phases[1] = None
    want = full.clone()
    want[:, 0::2, 1::2] = 0
    assert torch.equal(R.phase_interleave(phases, H, W), want)
    z = _rand(50, seed=16).double().requires_grad_(True)
    s = torch.sigmoid(z)
    G = _rand(50, seed=17).double()
    (s * G).sum().backward()
    _close(R.sigmoid_bwd(G, s.detach())["dz"], z.grad)


# ------------------------------------------------------------------------------------------------ Philox
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10"""
    got = R.philox4x32_10((0, 0), np.zeros((1, 4), np.uint32))[0]
    assert [f"{v:08x}" for v in got] == ["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"]
    got = R.philox4x32_10((0xa4093822, 0x299f31d0), np.array([[0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]], np.uint32))[0]
    assert [f"{v:08x}" for v in got] == ["d16cfe09", "94fdcceb", "5001e420", "24126ea1"]


def test_dropout_bits_follow_the_flat_index():
    p, seed = 0.3, (7 << 32) | 99
    whole = R.dropout_keep(seed, 2 ** 32 - 10, 7, 5, p)            # crosses the counter's high word
    assert np.array_equal(whole[2:], R.dropout_keep(seed, 2 ** 32 - 10 + 10, 5, 5, p))
    assert 0.5 < whole.mean() < 0.9
    assert not np.array_equal(whole, R.dropout_keep(seed + 1, 2 ** 32 - 10, 7, 5, p))
    assert R.dropout_keep(seed, 0, 3, 4, 0.0).all()


# ------------------------------------------------------------------------------------------------ refusals
@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libstp3_b200.so is not built")
    return _lib.lib()


F1 = 1 << 20            # a non-null pointer: never dereferenced, every call below is refused by its argument checks


def _refused(L, code, needle):
    assert code != 0
    msg = L.stp3_last_error().decode()
    assert needle in msg, msg


def test_refusals(L):
    big = 1 << 40
    _refused(L, L.stp3_conv_wgrad(None, 1, 8, 8, 64, 64, F1, 8, 8, 64, 64, 3, 3, 1, 1, 1, F1, big, F1, None), "null pointer")
    _refused(L, L.stp3_conv_wgrad(F1, 1, 8, 8, 64, 64, F1, 8, 8, 64, 64, 3, 3, 3, 1, 1, F1, big, F1, None), "stride")
    _refused(L, L.stp3_conv_wgrad(F1, 1, 8, 8, 64, 64, F1, 8, 8, 64, 64, 3, 3, 1, 1, 0, F1, big, F1, None), "dilation")
    _refused(L, L.stp3_conv_wgrad(F1, 1, 8, 8, 60, 64, F1, 8, 8, 64, 64, 3, 3, 1, 1, 1, F1, big, F1, None), "row stride")
    need = L.stp3_conv_wgrad_scratch_bytes(1, 8, 8, 64, 64, 3, 3, 1)
    assert need == R.wgrad_split(64, 9, 64, 64)[0] * 9 * 64 * 64 * 4
    _refused(L, L.stp3_conv_wgrad(F1, 1, 8, 8, 64, 64, F1, 8, 8, 64, 64, 3, 3, 1, 1, 1, F1, need - 1, F1, None), "scratch")
    _refused(L, L.stp3_conv3d_wgrad(F1, 1, 2, 8, 8, 64, 64, F1, 64, 64, 2, 3, 1, F1, big, F1, None), "square and odd")
    need3 = L.stp3_conv3d_wgrad_scratch_bytes(2, 3, 200, 200, 35, 35, 2, 3, 3)
    assert need3 == R.wgrad_split(240000, 18, 35, 35)[0] * 18 * 35 * 35 * 4
    _refused(L, L.stp3_conv3d_wgrad(F1, 2, 3, 200, 200, 35, 35, F1, 35, 35, 2, 3, 3, F1, need3 - 4, F1, None), "scratch")
    _refused(L, L.stp3_bn_stats(F1, 10, 4, 4, 1e-5, 0.1, F1, None, F1, F1, F1, F1, big, None), "running")
    _refused(L, L.stp3_bn_stats(F1, 10, 4, 4, 1e-5, 0.1, None, None, F1, F1, F1, F1, 8, None), "scratch")
    args = lambda **kw: dict(dict(x=F1, n=10, C=8, xcs=8, m=F1, s=F1, ga=F1, be=F1, r=None, rcs=0, relu=0, p=0.0,   # noqa: E731
                                  seed=0, off=0, y=F1, ycs=8, hi=None, lo=None, hlcs=0), **kw)
    apply = lambda a: L.stp3_bn_apply(*a.values(), None)            # noqa: E731
    _refused(L, apply(args(p=1.0)), "dropout p")
    _refused(L, apply(args(hi=F1)), "both bf16 planes")
    _refused(L, apply(args(hi=F1, lo=F1, hlcs=12)), "bf16 planes")
    _refused(L, apply(args(hi=F1 + 4, lo=F1, hlcs=64)), "bf16 planes")
    _refused(L, apply(args(ycs=4)), "fp32 output")
    _refused(L, L.stp3_bn_bwd_reduce(F1, 8, None, 0, F1, 8, None, F1, 10, 8, F1, F1, F1, big, None), "mean, invstd")
    _refused(L, L.stp3_bn_bwd_apply(F1, 8, None, 0, F1, 8, F1, F1, F1, F1, F1, 10, 8, F1, 4, None, 0, None), "row stride")
    _refused(L, L.stp3_image_channel_sums(F1, 65536, 4, 8, 8, F1, F1, big, None), "65535")
    _refused(L, L.stp3_upsample2x_window_f32(F1, 1, 2, 2, 8, F1, 12, 5, None), "outside rows")
    _refused(L, L.stp3_upsample2x_window_bwd(F1, 12, -1, 1, 2, 2, 8, F1, None), "outside rows")
    _refused(L, L.stp3_phase_interleave(F1, None, None, None, 1, 0, 4, 8, F1, None), "bad argument")
    _refused(L, L.stp3_sigmoid_bwd(F1, F1, 0, F1, None), "bad argument")
    _refused(L, L.stp3_temporal_pair_mean(F1, 1, 2, 8, 0, F1, None), "alias")
    assert L.stp3_conv_wgrad_scratch_bytes(1, 8, 8, 64, 64, 3, 3, 0) == 0
    assert L.stp3_bn_scratch_bytes(100, 8) == 100 * 2 * 8 * 8 and L.stp3_bn_scratch_bytes(1000, 8) == 128 * 2 * 8 * 8
