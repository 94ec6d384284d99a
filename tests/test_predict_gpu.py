"""GPU: the eval-mode prediction stage (N_FUTURE_FRAMES > 0) on sm_90a.

  - every kernel of csrc/predict_kernels.cu against an fp64 evaluation of its contract, on slots inside wider buffers:
    channels outside the slot and frames outside the call keep their sentinel bits;
  - every module against the fp64 oracle (oracle/torch_predict.py) at 48 x 64, B = 2, and against the reference's
    values (tests/golden/predict_modules_48x64.npz);
  - the whole Prediction model for the nuScenes and CARLA gate sets at 200 x 200, B = 1;
  - CUDA-graph replay and deterministic mode bitwise, and a perception model unaffected by a Prediction model that ran
    in the same process.
"""
import copy
import math
import os

import numpy as np
import pytest
import torch

from oracle import torch_dense as TD
from oracle import torch_predict as TP
from oracle.make_golden_predict import (_Stage, build_prediction_model, module_states, predict_cfg,
                                        predict_modules)
from stp3_b200 import dense
from stp3_b200.layers.convolutions import DeepLabHead
from stp3_b200.utils import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SENT = 7.25          # sentinel value of every channel a call must not write (exact in bf16; lo plane 0)


# ------------------------------------------------------------------------------------------------ helpers
def rand_hl(B, T, H, W, cs, gen, scale=1.0, offset=0.0):
    """HL whose hi/lo planes hold a random fp32 tensor; value(hl) is its exact fp64 value."""
    x = torch.randn((B, T, H, W, cs), generator=gen, device=DEV) * scale + offset
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return dense.HL(hi.contiguous(), lo.contiguous(), cs)


def sentinel_hl(B, T, H, W, cs):
    return dense.HL(torch.full((B, T, H, W, cs), SENT, dtype=torch.bfloat16, device=DEV),
                    torch.zeros((B, T, H, W, cs), dtype=torch.bfloat16, device=DEV), cs)


def value(h):
    return h.hi.double() + h.lo.double()


def assert_close(got, ref, bar_rel=2e-5, bar_max=2e-6, what=""):
    """|got - ref| <= bar_rel |ref| + bar_max max|ref|: an fp32 evaluation stored as hi/lo (2^-17 relative)."""
    mx = ref.abs().max().item()
    err = (got - ref).abs()
    lim = bar_rel * ref.abs() + bar_max * max(mx, 1e-30)
    bad = (err > lim)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, worst {err.max().item():.3e} (max|ref| {mx:.3e})"


def untouched(out_before_hi, out_before_lo, out, keep_mask):
    """Channels / frames outside the written slot keep their bits."""
    assert torch.equal(out.hi[keep_mask], out_before_hi[keep_mask]) and torch.equal(out.lo[keep_mask], out_before_lo[keep_mask])


SIZES = [(13, 13), (25, 25), (48, 64), (200, 200)]
IMAGES = [1, 14]


def shapes():
    for H, W in SIZES:
        for n in IMAGES:
            yield pytest.param(H, W, n, id=f"{H}x{W}-n{n}")


def _mask(shape, coff, C, frames=None):
    """True where a call over channels [coff, coff + C) (and frames [t0, t0+T)) must NOT write."""
    m = torch.ones(shape, dtype=torch.bool, device=DEV)
    if frames is None:
        m[..., coff:coff + C] = False
    else:
        t0, T = frames
        m[:, t0:t0 + T, ..., coff:coff + C] = False
    return m


# ------------------------------------------------------------------------------------------------ kernel contracts
@pytest.mark.parametrize("H, W, n", list(shapes()))
@pytest.mark.parametrize("C, cs, coff", [(64, 64, 0), (64, 192, 64), (96, 128, 32)])
def test_gru_kernels_contract(H, W, n, C, cs, coff):
    """stp3_gru_gates, stp3_gru_update (two destinations, one of them a frame slot) and stp3_hl_copy /
    stp3_hl_broadcast, against fp64."""
    gen = torch.Generator(device=DEV).manual_seed(H * 1000 + n + C)
    B, T = (2, n // 2) if n > 1 else (1, 1)
    g = rand_hl(B, T, H, W, 2 * cs, gen, 2.0)                      # [u | r] at coff and cs + coff
    h = rand_hl(B, T, H, W, cs, gen)
    ht = rand_hl(B, T, H, W, cs, gen)
    u, r = value(g)[..., coff:coff + C], value(g)[..., cs + coff:cs + coff + C]
    hv, tv = value(h)[..., coff:coff + C], value(ht)[..., coff:coff + C]
    out = sentinel_hl(B, T, H, W, cs)
    b_hi, b_lo = out.hi.clone(), out.lo.clone()
    dense.gru_gates((g, cs + coff), (h, coff), (out, coff), C)
    assert_close(value(out)[..., coff:coff + C], (1 - torch.sigmoid(r)) * hv, what="gru_gates")
    untouched(b_hi, b_lo, out, _mask(out.hi.shape, coff, C))
    # update into a slot and into frames [1, 1 + T) of a (B, T + 2) stack
    stack = sentinel_hl(B, T + 2, H, W, cs)
    s_hi, s_lo = stack.hi.clone(), stack.lo.clone()
    out = sentinel_hl(B, T, H, W, cs)
    dense.gru_update((g, coff), (h, coff), (ht, coff), (out, coff), C, out2=(stack, coff, 1))
    s = torch.sigmoid(u)
    ref = (1 - s) * hv + s * tv
    assert_close(value(out)[..., coff:coff + C], ref, what="gru_update")
    assert torch.equal(stack.hi[:, 1:1 + T, ..., coff:coff + C], out.hi[..., coff:coff + C])
    untouched(s_hi, s_lo, stack, _mask(stack.hi.shape, coff, C, (1, T)))
    # in place: out is h itself
    h2 = dense.HL(h.hi.clone(), h.lo.clone(), cs)
    dense.gru_update((g, coff), (h2, coff), (ht, coff), (h2, coff), C)
    assert torch.equal(h2.hi[..., coff:coff + C], out.hi[..., coff:coff + C])
    assert torch.equal(h2.lo[..., coff:coff + C], out.lo[..., coff:coff + C])
    # copies are exact
    cp = sentinel_hl(B, T, H, W, cs)
    dense.hl_copy((h, coff), (cp, coff), C)
    assert torch.equal(cp.hi[..., coff:coff + C], h.hi[..., coff:coff + C])
    assert torch.equal(cp.lo[..., coff:coff + C], h.lo[..., coff:coff + C])
    vec = torch.randn((B * T, C + 8), generator=gen, device=DEV)
    bc = sentinel_hl(B, T, H, W, cs)
    c_hi, c_lo = bc.hi.clone(), bc.lo.clone()
    dense.hl_broadcast(vec, (bc, coff), C)
    want = vec[:, :C].double().view(B, T, 1, 1, C).expand(B, T, H, W, C)
    assert_close(value(bc)[..., coff:coff + C], want, bar_rel=2 ** -16, bar_max=0, what="hl_broadcast")
    untouched(c_hi, c_lo, bc, _mask(bc.hi.shape, coff, C))


def ln64(x, gamma, beta, eps):
    u = x.mean(-1, keepdim=True)
    v = ((x - u) ** 2).mean(-1, keepdim=True)
    return (x - u) / torch.sqrt(v + eps) * gamma.double() + beta.double()


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


@pytest.mark.parametrize("H, W, n", list(shapes()))
@pytest.mark.parametrize("C, cs, coff", [(64, 64, 0), (64, 192, 64), (96, 128, 32), (256, 256, 0)])
def test_norm_act_and_mix_contract(H, W, n, C, cs, coff):
    """stp3_channel_norm_act (LN + GELU, + GELU(y), GELU alone in place) and stp3_trust_mix against fp64."""
    gen = torch.Generator(device=DEV).manual_seed(H * 7 + n + C)
    B, T = (2, n // 2) if n > 1 else (1, 1)
    x = rand_hl(B, T, H, W, cs, gen, 3.0)
    y = rand_hl(B, T, H, W, cs, gen)
    gamma = 1 + 0.25 * torch.randn(C, generator=gen, device=DEV)
    beta = 0.25 * torch.randn(C, generator=gen, device=DEV)
    xv, yv = value(x)[..., coff:coff + C], value(y)[..., coff:coff + C]
    out = sentinel_hl(B, T, H, W, cs)
    b_hi, b_lo = out.hi.clone(), out.lo.clone()
    dense.channel_norm_act((x, coff), (out, coff), C, ln=(gamma, beta, 1e-6), gelu=True, y=(y, coff), gelu_y=True)
    assert_close(value(out)[..., coff:coff + C], gelu64(ln64(xv, gamma, beta, 1e-6)) + gelu64(yv), what="norm_act")
    untouched(b_hi, b_lo, out, _mask(out.hi.shape, coff, C))
    dense.channel_norm_act((x, coff), (out, coff), C, ln=(gamma, beta, 1e-6), y=(y, coff))
    assert_close(value(out)[..., coff:coff + C], ln64(xv, gamma, beta, 1e-6) + yv, what="norm + y")
    x2 = dense.HL(x.hi.clone(), x.lo.clone(), cs)
    dense.channel_norm_act((x2, coff), (x2, coff), C, gelu=True)
    assert_close(value(x2)[..., coff:coff + C], gelu64(xv), what="gelu in place")
    # trust mix: t, s1, s2 slots of one buffer, three destinations
    w = torch.randn((2, C), generator=gen, device=DEV) * 0.3
    src = rand_hl(B, T, H, W, 3 * cs, gen)
    tv, s1, s2 = (value(src)[..., k * cs + coff:k * cs + coff + C] for k in range(3))
    z = torch.einsum("kc,...c->...k", w.double(), tv)
    p = torch.softmax(z, -1)
    ref = s2 * p[..., 0:1] + s1 * p[..., 1:2]
    d1, d2 = sentinel_hl(B, T, H, W, cs), sentinel_hl(B, T + 1, H, W, cs)
    h1, l1, h2, l2 = d1.hi.clone(), d1.lo.clone(), d2.hi.clone(), d2.lo.clone()
    dense.trust_mix((src, coff), w, (src, cs + coff), (src, 2 * cs + coff), [(d1, coff), (d2, coff, 1)], C)
    assert_close(value(d1)[..., coff:coff + C], ref, what="trust_mix")
    assert torch.equal(d2.hi[:, 1:, ..., coff:coff + C], d1.hi[..., coff:coff + C])
    untouched(h1, l1, d1, _mask(d1.hi.shape, coff, C))
    untouched(h2, l2, d2, _mask(d2.hi.shape, coff, C, (1, T)))


@pytest.mark.parametrize("H, W, n", list(shapes()))
@pytest.mark.parametrize("C, cs, coff", [(64, 64, 0), (64, 192, 64), (96, 128, 32)])
def test_dw_ln_and_maxpool_contract(H, W, n, C, cs, coff):
    """stp3_dw_ln (depthwise 7x7 + bias + LN) and stp3_maxpool2_pad against fp64 (F.conv2d / F.pad + max_pool2d)."""
    import torch.nn.functional as F
    gen = torch.Generator(device=DEV).manual_seed(H * 13 + n + C)
    B, T = (2, n // 2) if n > 1 else (1, 1)
    x = rand_hl(B, T, H, W, cs, gen)
    w = torch.randn((49, C), generator=gen, device=DEV) * 0.2
    b = torch.randn(C, generator=gen, device=DEV) * 0.1
    gamma = 1 + 0.25 * torch.randn(C, generator=gen, device=DEV)
    beta = 0.25 * torch.randn(C, generator=gen, device=DEV)
    xv = value(x)[..., coff:coff + C].reshape(B * T, H, W, C).permute(0, 3, 1, 2)
    conv = F.conv2d(xv, w.double().t().reshape(C, 1, 7, 7), b.double(), padding=3, groups=C).permute(0, 2, 3, 1)
    ref = ln64(conv, gamma, beta, 1e-6).reshape(B, T, H, W, C)
    out = sentinel_hl(B, T, H, W, cs)
    b_hi, b_lo = out.hi.clone(), out.lo.clone()
    dense.dw_ln((x, coff), w, b, 7, (gamma, beta, 1e-6), (out, coff), C)
    assert_close(value(out)[..., coff:coff + C], ref, bar_rel=2e-5, bar_max=1e-5, what="dw_ln")
    untouched(b_hi, b_lo, out, _mask(out.hi.shape, coff, C))
    # max pool over every channel of the buffer (its padding included); negative inputs show the padded zeros
    xm = rand_hl(B, T, H, W, cs, gen, offset=-1.0)   # mostly negative: the padded zeros win the odd edges
    mp = dense.maxpool2_pad(xm)
    xmv = value(xm).reshape(B * T, H, W, cs).permute(0, 3, 1, 2)
    want = F.max_pool2d(F.pad(xmv, (0, W % 2, 0, H % 2), value=0), 2).permute(0, 2, 3, 1)
    got = value(mp).reshape(want.shape)
    assert torch.equal(got, want)


def test_padding_channels_stay_zero():
    """C = 40 real channels of 64-channel buffers: the padding channels [40, 64) of every output come out +0 in both
    planes (the outputs start zeroed, as the modules allocate the buffers whose padding a convolution reads), while the
    inputs carry nonzero padding that no result may pick up (LayerNorm statistics, the mix's dot products, the taps)."""
    import torch.nn.functional as F
    gen = torch.Generator(device=DEV).manual_seed(40)
    B, T, H, W, C, cs = 2, 1, 25, 25, 40, 64
    zero = lambda c=cs: dense.HL.zeros(B, T, H, W, C, DEV, cp=c)

    def pad_zero(h, c=C):
        assert not h.hi[..., c:].any() and not h.lo[..., c:].any(), "padding channels written"
        assert not torch.signbit(h.hi[..., c:].float()).any()

    x, hh, ht = rand_hl(B, T, H, W, cs, gen), rand_hl(B, T, H, W, cs, gen), rand_hl(B, T, H, W, cs, gen)
    g = rand_hl(B, T, H, W, 2 * cs, gen)
    xv, hv, tv = value(x)[..., :C], value(hh)[..., :C], value(ht)[..., :C]
    out = zero()
    dense.gru_gates((g, cs), hh, out, C)
    pad_zero(out)
    assert_close(value(out)[..., :C], (1 - torch.sigmoid(value(g)[..., cs:cs + C])) * hv, what="gru_gates")
    out = zero()
    dense.gru_update(g, hh, ht, out, C)
    pad_zero(out)
    su = torch.sigmoid(value(g)[..., :C])
    assert_close(value(out)[..., :C], (1 - su) * hv + su * tv, what="gru_update")
    gamma = 1 + 0.25 * torch.randn(C, generator=gen, device=DEV)
    beta = 0.25 * torch.randn(C, generator=gen, device=DEV)
    out = zero()
    dense.channel_norm_act(x, out, C, ln=(gamma, beta, 1e-6), gelu=True, y=hh, gelu_y=True)
    pad_zero(out)
    assert_close(value(out)[..., :C], gelu64(ln64(xv, gamma, beta, 1e-6)) + gelu64(hv), what="norm_act")
    w = torch.randn((49, C), generator=gen, device=DEV) * 0.2
    b = torch.randn(C, generator=gen, device=DEV) * 0.1
    out = zero()
    dense.dw_ln(x, w, b, 7, (gamma, beta, 1e-6), out, C)
    pad_zero(out)
    conv = F.conv2d(xv.reshape(B * T, H, W, C).permute(0, 3, 1, 2), w.double().t().reshape(C, 1, 7, 7), b.double(),
                    padding=3, groups=C).permute(0, 2, 3, 1).reshape(B, T, H, W, C)
    assert_close(value(out)[..., :C], ln64(conv, gamma, beta, 1e-6), bar_max=1e-5, what="dw_ln")
    w2 = torch.randn((2, C), generator=gen, device=DEV) * 0.3
    out = zero()
    dense.trust_mix(x, w2, hh, ht, [out], C)
    pad_zero(out)
    p = torch.softmax(torch.einsum("kc,...c->...k", w2.double(), xv), -1)
    assert_close(value(out)[..., :C], tv * p[..., :1] + hv * p[..., 1:], what="trust_mix")
    out = zero()
    dense.hl_copy(x, out, C)
    pad_zero(out)
    out = zero()
    dense.hl_broadcast(torch.randn((B * T, cs), generator=gen, device=DEV), out, C)
    pad_zero(out)
    xm = dense.HL(x.hi.clone(), x.lo.clone(), C)          # the max pool runs over the whole stride: zero padding in
    xm.hi[..., C:] = 0
    xm.lo[..., C:] = 0
    pad_zero(dense.maxpool2_pad(xm))
    # a module whose real channels do not fill the stride: the distribution's Bottlenecks (32 and 16 channels)
    m = predict_modules().to(DEV)
    y = dense.from_f32(torch.randn((B, 1, 64, 50, 50), generator=gen, device=DEV))
    for blk, c in zip(m.present_distribution.encoder.model, (32, 32, 32, 32)):
        y = blk.forward_hl(y)
        pad_zero(y, c)


def test_slot_checks():
    """A slot whose buffer has another batch or map size than the call is refused before any launch, and so is a
    stp3_dw_ln output whose address span overlaps its input's (here: other channels of the same buffer)."""
    gen = torch.Generator(device=DEV).manual_seed(1)
    a, small = rand_hl(2, 1, 25, 25, 64, gen), rand_hl(1, 1, 25, 25, 64, gen)
    narrow = rand_hl(2, 1, 25, 24, 64, gen)
    for bad in (small, narrow):
        with pytest.raises(AssertionError):
            dense.gru_gates(a, a, bad, 64)
        with pytest.raises(AssertionError):
            dense.trust_mix(a, torch.zeros((2, 64), device=DEV), a, a, [a, bad], 64)
    two = rand_hl(2, 1, 25, 25, 128, gen)
    w = torch.zeros((49, 64), device=DEV)
    v = torch.ones(64, device=DEV)
    with pytest.raises(RuntimeError, match="overlap"):
        dense.dw_ln((two, 0), w, v, 7, (v, v, 1e-6), (two, 64), 64)


def test_layer_norm_standalone():
    """The drop-in LayerNorm called on its own, both data formats, against fp64."""
    from stp3_b200.layers.convolutions import LayerNorm
    gen = torch.Generator(device=DEV).manual_seed(2)
    for fmt, shape in (("channels_first", (3, 64, 13, 17)), ("channels_last", (3, 13, 17, 64))):
        ln = LayerNorm(64, eps=1e-6, data_format=fmt).to(DEV).eval()
        with torch.no_grad():
            ln.weight.copy_(1 + 0.25 * torch.randn(64, generator=gen, device=DEV))
            ln.bias.copy_(0.25 * torch.randn(64, generator=gen, device=DEV))
        x = torch.randn(shape, generator=gen, device=DEV) * 3
        y = ln(x)
        if fmt == "channels_first":
            ref = TP.layer_norm_cf(x.double(), ln)
        else:
            ref = torch.nn.functional.layer_norm(x.double(), (64,), ln.weight.double(), ln.bias.double(), 1e-6)
        assert y.shape == x.shape
        check(f"LayerNorm {fmt}", y, ref, 1e-5)


# ------------------------------------------------------------------------------------------------ modules
@pytest.fixture(scope="module")
def mods():
    m = predict_modules().to(DEV)
    return m, copy.deepcopy(m).double()


def rel_to_max(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def check(what, got, ref, bar):
    d = rel_to_max(got, ref)
    print(f"  {what:28s} {d:.2e} of max vs fp64 (bar {bar:.0e})")
    assert d < bar, (what, d)


MODULE_BAR = 3e-4


def test_bottleneck_odd_sizes(mods):
    """The 25 -> 13 and 13 -> 7 steps take the odd-size pad (present distribution at 200^2)."""
    m, m64 = mods
    gen = torch.Generator(device=DEV).manual_seed(3)
    for H, W in ((25, 25), (13, 7), (48, 64)):
        x = torch.randn((2, 64, H, W), generator=gen, device=DEV)
        got = m.present_distribution.encoder.model[0](x)
        ref = TP.bottleneck(x.double(), m64.present_distribution.encoder.model[0])
        assert got.shape == ref.shape == (2, 32, (H + 1) // 2, (W + 1) // 2)
        check(f'Bottleneck {H}x{W}', got, ref, MODULE_BAR)


def test_distribution_module(mods):
    m, m64 = mods
    s = module_states().to(DEV)
    got = m.present_distribution(s[:, -1:])
    ref = TP.distribution(s[:, -1:].double(), m64.present_distribution)
    check('DistributionModule', got, ref, MODULE_BAR)
    g = np.load(os.path.join(GOLD, "predict_modules_48x64.npz"))
    d = np.abs(got.double().cpu().numpy().reshape(-1)[g["mu_log_sigma_index"]] - g["mu_log_sigma_ref"]).max()
    assert d / float(g["mu_log_sigma_max"]) < 1e-3


def test_block_and_bottleblock(mods):
    m, m64 = mods
    gen = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn((2, 64, 48, 64), generator=gen, device=DEV)
    blk = m.future_prediction.res_blocks1[0]
    check('Block', blk(x), TP.block(x.double(), m64.future_prediction.res_blocks1[0]), MODULE_BAR)
    x2 = torch.randn((2, 128, 48, 64), generator=gen, device=DEV)
    bb = m.future_prediction.dual_grus.trusting_gate[0]
    check('Bottleblock', bb(x2), TP.bottleblock(x2.double(), m64.future_prediction.dual_grus.trusting_gate[0]), MODULE_BAR)


def test_spatial_gru(mods):
    m, m64 = mods
    s = module_states().to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(6)
    h0 = torch.randn((2, 64, 48, 64), generator=gen, device=DEV)
    for i in range(2):
        got = m.future_prediction.spatial_grus[i](s, h0)
        ref = TP.spatial_gru(s.double(), h0.double(), m64.future_prediction.spatial_grus[i])
        check(f'SpatialGRU {i}', got, ref, MODULE_BAR)


def test_dual_gru_and_future_prediction(mods):
    m, m64 = mods
    s = module_states().to(DEV)
    mu = TP.distribution(s[:, -1:].double(), m64.present_distribution)[:, :, :32]
    x64 = mu.view(2, 1, 32, 1, 1).expand(2, 1, 32, 48, 64)
    got = m.future_prediction.dual_grus(x64.float(), s)
    check('Dual_GRU', got, TP.dual_gru(x64, s.double(), m64.future_prediction.dual_grus), MODULE_BAR)
    got = m.future_prediction(x64.float(), s)
    ref = TP.future_prediction(x64, s.double(), m64.future_prediction)
    assert got.shape == (2, 7, 64, 48, 64)
    check('FuturePrediction', got, ref, MODULE_BAR)
    # the whole stage from the states (distribution included) against the reference's fp32 values
    for prob, name in ((True, "modules_48x64"), (False, "noprob_48x64")):
        gm = predict_modules(probabilistic=prob).to(DEV)
        hl = dense.from_f32(s)
        x = None
        if prob:
            mls = gm.present_distribution.forward_hl(dense.from_f32(s[:, -1:].contiguous()))
            x = dense.HL.empty(2, 1, 48, 64, 32, DEV)
            dense.hl_broadcast(mls, x, 32)
        y = dense.to_f32(gm.future_prediction.forward_hl(x, hl), 0, 64)
        ref = TP.predict_stage(s.double(), _Stage(copy.deepcopy(gm).double(), prob))
        check(name, y, ref, MODULE_BAR)
        g = np.load(os.path.join(GOLD, f"predict_{name}.npz"))
        d = np.abs(y.double().cpu().numpy().reshape(-1)[g["future_index"]] - g["future_ref"]).max()
        assert d / float(g["future_max"]) < 1e-3, name


# ------------------------------------------------------------------------------------------------ whole model
def _run(model, inp):
    with torch.no_grad():
        return model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                      inp["extrinsics"], inp["future_egomotion"])


def _f32(v):
    """An HL as fp32 (B, T, 64, H, W)."""
    return dense.to_f32(v, 0, 64)


def _nchw(v64):
    """(B, 1, H, W, C) channels-last fp64 -> (B, C, H, W)."""
    return v64[:, 0].permute(0, 3, 1, 2)


class _Recorder:
    """Checks, launch group by launch group, what the Prediction model computes against fp64 fed with the inputs the
    model itself produced: every conv-GRU cell step (temporal._gru_step), every trusting-gate mix (dense.trust_mix),
    every Bottleblock, Block and DeepLab head call, and the present distribution."""

    def __init__(self, model, m64, monkeypatch):
        from stp3_b200.layers import temporal
        self.worst, self.outputs, self.wiring = {}, {}, {}
        fp, fp64 = model.future_prediction, m64.future_prediction
        cells = {}
        dg, dg64 = fp.dual_grus, fp64.dual_grus
        P = dg.packed()
        cells[id(P["gate1"])] = ("Dual_GRU cell 1", dg64.conv_update_1, dg64.conv_reset_1, dg64.conv_state_tilde_1, 32)
        cells[id(P["gate2"])] = ("Dual_GRU cell 2", dg64.conv_update_2, dg64.conv_reset_2, dg64.conv_state_tilde_2, 64)
        for i, (g, g64) in enumerate(zip(fp.spatial_grus, fp64.spatial_grus)):
            cells[id(g.packed()["gate"])] = (f"SpatialGRU {i} cell", g64.conv_update, g64.conv_reset,
                                             g64.conv_state_tilde, 64)
        orig_step, orig_mix = temporal._gru_step, dense.trust_mix

        def step(buf, gate, prop, out2=None):
            before = value(buf)
            orig_step(buf, gate, prop, out2)
            name, cu, cr, ct, nin = cells[id(gate)]
            ref = TP._gru_cell(_nchw(before[..., 64:64 + nin]), _nchw(before[..., :64]), cu, cr, ct)
            self.note(name, _nchw(value(buf)[..., :64]), ref)

        def mix(t, w, s1, s2, dsts, C, T=None):
            tv, v1, v2 = value(t)[..., :C], value(s1[0])[..., s1[1]:s1[1] + C], value(s2[0])[..., s2[1]:s2[1] + C]
            orig_mix(t, w, s1, s2, dsts, C, T)
            p = torch.softmax(torch.einsum("kc,...c->...k", w.double(), tv), -1)
            d = dsts[0]
            self.note("trusting-gate mix", value(d[0])[..., d[1]:d[1] + C], v2 * p[..., :1] + v1 * p[..., 1:])

        monkeypatch.setattr(temporal, "_gru_step", step)
        monkeypatch.setattr(dense, "trust_mix", mix)

        def wrap(mod, mod64, name, fn, cin):
            orig = mod.forward_hl

            def f(x):
                xin = dense.to_f32(x, 0, cin).double()
                y = orig(x)
                b, s = xin.shape[:2]
                ref = fn(xin.reshape(b * s, *xin.shape[2:]), mod64)
                self.outputs[name] = dense.to_f32(y, 0, ref.shape[1])
                self.note(name, self.outputs[name].reshape(b * s, *ref.shape[1:]), ref)
                return y
            monkeypatch.setattr(mod, "forward_hl", f)

        wrap(dg.trusting_gate[0], dg64.trusting_gate[0], "Bottleblock", TP.bottleblock, 128)
        for blk, blk64 in list(zip(fp.res_blocks1, fp64.res_blocks1)) + list(zip(fp.res_blocks[0], fp64.res_blocks[0])):
            wrap(blk, blk64, "Block", TP.block, 64)
        wrap(fp.res_blocks[1], fp64.res_blocks[1], "DeepLabHead", TD.deeplab_head, 64)
        pd, pd64 = model.present_distribution, m64.present_distribution
        orig_pd = pd.forward_hl

        def dist(x):
            y = orig_pd(x)
            self.wiring["distribution_in"], self.wiring["mu_log_sigma"] = dense.to_f32(x, 0, 64), y.clone()
            self.note("DistributionModule", y, TP.distribution(dense.to_f32(x, 0, 64).double(), pd64)[:, 0])
            return y
        monkeypatch.setattr(pd, "forward_hl", dist)
        orig_dual = dg.forward_hl

        def dual(x, state, out, out_t0=0):
            self.wiring["latent"], self.wiring["dual_state"] = dense.to_f32(x, 0, 32), dense.to_f32(state, 0, 64)
            return orig_dual(x, state, out, out_t0)
        monkeypatch.setattr(dg, "forward_hl", dual)
        self.future = None
        orig_dec = model.decoder.forward_hl

        def dec(x):
            self.future = dense.to_f32(x, 0, 64)
            return orig_dec(x)
        monkeypatch.setattr(model.decoder, "forward_hl", dec)

    def note(self, name, got, ref):
        self.worst[name] = max(self.worst.get(name, 0.0), rel_to_max(got, ref))


OUT_KEYS = ("segmentation", "pedestrian", "hdmap", "instance_center", "instance_offset", "instance_flow")
STEP_BAR = 3e-4
CHAIN_FACTOR = 2.0        # chained distance to fp64 over the reference fp32's own (see the end-to-end test)


@pytest.mark.parametrize("carla", [False, True], ids=["nuscenes", "carla"])
def test_prediction_model_end_to_end(carla, monkeypatch):
    """The Prediction model at 200 x 200, B = 1, from the lift-splat to every decoder head.

    Launch group by launch group -- every conv-GRU cell step of the Dual_GRU warm-up, of its four future steps and of
    both SpatialGRUs, every trusting-gate mix, Bottleblock, Block and the DeepLab head, the present distribution and
    the decoder, each fed the inputs the model itself produced -- the outputs sit within 3e-4 of max of fp64.  The
    present states (the temporal model's output) and the present-frame hdmap sit within 1e-3 of max of the reference's
    fp32 values.

    Between the launch groups the hand-offs are checked exactly: the distribution reads frame S - 1 of the present
    states, the Dual_GRU's latent input is mu (not log sigma) broadcast over the map and its state input is the present
    states, and the decoder reads the DeepLab head's output.

    Chained through the recurrences, the distance to fp64 is a property of these synthetic weights: in fp64 they
    amplify a 1e-6 relative perturbation of the present states to 2.4e-4 over the four Dual_GRU steps alone, and the
    reference's own fp32 run ends 2e-2 of max from fp64 on the predicted frames (the fixture's `fulldev`, one value per
    output).  This build lands at the same order (1.9-2.4e-2 on the frames over four runs; the tiling the autotuner
    picks changes the last bits and the recurrence amplifies them), so the chained frames and every decoder output are
    held to CHAIN_FACTOR times the reference's own distance: room for that run-to-run spread, while a wiring error, which
    moves the outputs by O(1) of max, fails."""
    cfg = predict_cfg(carla)
    model = build_prediction_model(cfg).to(DEV)
    m64 = copy.deepcopy(model).double()
    inp = syn.lift_inputs(syn.CONFIGS["perceive"], 1, seed=0)
    _run(model, inp)                                  # packs the weights the recorder keys on
    rec = _Recorder(model, m64, monkeypatch)
    states = {}
    orig = model._predict_hl
    monkeypatch.setattr(model, "_predict_hl", lambda st: (states.setdefault("states", _f32(st)), orig(st))[1])
    out = _run(model, inp)
    g = np.load(os.path.join(GOLD, f"predict_e2e_{'carla' if carla else 'nuscenes'}.npz"))
    with torch.no_grad():
        out64 = TD.decoder(rec.future.double(), m64.decoder)
        for k in OUT_KEYS:
            if out.get(k) is None:
                continue
            if k == "instance_center":
                # a sigmoid head: its outputs move by at most 1/4 of the logits' error, so the error is taken
                # relative to a quarter of the fp64 logits' max
                dec = copy.deepcopy(m64.decoder)
                dec.instance_center_head = dec.instance_center_head[:4]
                scale = 0.25 * TD.decoder(rec.future.double(), dec)[k].abs().max().item()
                rec.worst[f"decoder {k} (logit scale)"] = (out[k].double() - out64[k]).abs().max().item() / scale
            else:
                rec.note(f"decoder {k}", out[k], out64[k])
        fut64 = TP.predict_stage(states["states"].double(), m64)
        chained = TD.decoder(fut64, m64.decoder)
    assert rec.future.shape == (1, 7, 64, 200, 200)
    expected = {"Dual_GRU cell 1", "Dual_GRU cell 2", "SpatialGRU 0 cell", "SpatialGRU 1 cell", "trusting-gate mix",
                "Bottleblock", "Block", "DeepLabHead", "DistributionModule"}
    assert expected <= set(rec.worst), set(rec.worst)
    for name, d in sorted(rec.worst.items()):
        print(f"  {name:28s} {d:.2e} of max vs fp64 on its own inputs (bar {STEP_BAR:.0e})")
    print(f"  chained future frames        {rel_to_max(rec.future, fut64):.2e} of max vs fp64 "
          f"(reference fp32: {float(g['future_fulldev']):.2e})")
    for k in OUT_KEYS:
        if out.get(k) is not None:
            print(f"  chained {k:20s} {rel_to_max(out[k], chained[k]):.2e} of max vs fp64 "
                  f"(reference fp32: {float(g[f'{k}_fulldev']):.2e})")
    for k, t in (("states", states["states"]), ("hdmap", out.get("hdmap"))):
        if t is None:
            continue
        d = np.abs(t.double().cpu().numpy().reshape(-1)[g[f"{k}_index"]] - g[f"{k}_ref"]).max() / float(g[f"{k}_max"])
        print(f"  {k:28s} {d:.2e} of max vs the reference (bar 1e-03)")
        assert d < 1e-3, (k, d)
    for name, d in rec.worst.items():
        assert d < STEP_BAR, (name, d)
    # hand-offs between the launch groups
    w, st = rec.wiring, states["states"]
    assert torch.equal(w["distribution_in"], st[:, -1:])
    assert torch.equal(w["dual_state"], st)
    mu = w["mu_log_sigma"][:, :32].double().view(1, 1, 32, 1, 1).expand(w["latent"].shape)
    assert (w["latent"].double() - mu).abs().max() <= 2 ** -16 * mu.abs().max()
    assert torch.equal(rec.future, rec.outputs["DeepLabHead"])
    # the chain
    chain = {"future": rel_to_max(rec.future, fut64)}
    chain.update({k: rel_to_max(out[k], chained[k]) for k in OUT_KEYS if out.get(k) is not None})
    for k, d in chain.items():
        bar = CHAIN_FACTOR * float(g[f"{k}_fulldev"])
        assert d < bar, (k, d, bar)


def test_predict_hl_through_stp3():
    """STP3._predict_hl itself -- the copy of frame S - 1 into the distribution, mu into the latent slot, the future
    prediction -- on the 48 x 64, B = 2 module states, where the chain is not amplified: within the module bar of the
    fp64 stage and 1e-3 of max of the reference's values.  The model's weights are the fixture's (init_exact keyed by
    the same state-dict names)."""
    s = module_states().to(DEV)
    for prob, name in ((True, "modules_48x64"), (False, "noprob_48x64")):
        cfg = predict_cfg(False)
        cfg.PROBABILISTIC.ENABLED = prob
        model = build_prediction_model(cfg).to(DEV)
        sd = model.state_dict()
        for k, v in predict_modules(probabilistic=prob).state_dict().items():
            assert torch.equal(sd[k].cpu(), v), k
        y = dense.to_f32(model._predict_hl(dense.from_f32(s)), 0, 64)
        ref = TP.predict_stage(s.double(), copy.deepcopy(model).double())
        check(f"STP3._predict_hl {name}", y, ref, MODULE_BAR)
        g = np.load(os.path.join(GOLD, f"predict_{name}.npz"))
        d = np.abs(y.double().cpu().numpy().reshape(-1)[g["future_index"]] - g["future_ref"]).max()
        assert d / float(g["future_max"]) < 1e-3, name


def test_graph_replay_and_deterministic_mode_are_bitwise():
    from stp3_b200.models.stp3 import GraphedPerception
    cfg = predict_cfg(False)
    model = build_prediction_model(cfg).to(DEV)
    inp = syn.lift_inputs(syn.CONFIGS["perceive"], 1, seed=1)
    torch.use_deterministic_algorithms(True)
    try:
        a = _run(model, inp)
        a = {k: v.clone() for k, v in a.items() if torch.is_tensor(v)}
        b = _run(model, inp)
        for k in a:
            assert torch.equal(a[k], b[k]), k
        g = GraphedPerception(model, 1, 6)
        with torch.no_grad():
            o = g(inp["feat"], inp["depth_logits"], inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        torch.cuda.synchronize()
        for k in a:
            if k != "depth_prediction":
                assert torch.equal(a[k], o[k]), k
        assert a["instance_flow"].shape[1] == 7
    finally:
        torch.use_deterministic_algorithms(False)


def test_perception_model_unaffected_by_a_prediction_model():
    import bench
    torch.use_deterministic_algorithms(True)
    try:
        perc = bench.build_model(DEV)
        inp = syn.lift_inputs(syn.CONFIGS["perceive"], 1, seed=2)
        before = {k: v.clone() for k, v in _run(perc, inp).items() if torch.is_tensor(v)}
        pred = build_prediction_model(predict_cfg(False)).to(DEV)
        _run(pred, inp)
        after = _run(perc, inp)
        for k in before:
            assert torch.equal(before[k], after[k]), k
    finally:
        torch.use_deterministic_algorithms(False)
