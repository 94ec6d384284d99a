"""CPU: the float64 reference of the trunk and helper entry points (tests/aux_reference.py) against PyTorch's own
definitions of the same operations, the squeeze-excite weight layout against the library's size query, the argument
refusals of the nine entry points (they return before any CUDA call, so they run without a device), and a guard that
every call of them goes through the dense wrappers the GPU contract test records."""
import ast
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import _lib, dense, dense_train
from tests import aux_reference as R


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).float() * scale


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    assert float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-300), float((a - b).abs().max())


def _planes(x_cl, cs, junk_seed=None):
    """(N, H, W, C) fp32 -> hi/lo planes (N, H, W, cs); channels [C, cs) hold junk when junk_seed is given"""
    N, H, W, C = x_cl.shape
    full = torch.zeros(N, H, W, cs)
    full[..., :C] = x_cl
    if junk_seed is not None:
        full[..., C:] = _rand(N, H, W, cs - C, seed=junk_seed, scale=1e3)
    return R.split(full)


# ------------------------------------------------------------------------------------------------ bf16 rounding
def test_bf16_rounding_is_torchs():
    g = torch.Generator().manual_seed(1)
    bits = torch.randint(-2 ** 31, 2 ** 31, (200000,), generator=g, dtype=torch.int64).to(torch.int32)
    x = bits.view(torch.float32)
    x = x[torch.isfinite(x)]
    special = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, 3.3895314e38, 3.3961e38, -3.4028235e38,
                            1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -8 + 2 ** -20], dtype=torch.float32)
    x = torch.cat([x, special])
    assert torch.equal(R.bf16_rn(x).view(torch.int16), x.to(torch.bfloat16).view(torch.int16))
    hi, lo = R.split(x)
    assert torch.equal(lo.view(torch.int16), (x - x.to(torch.bfloat16).float()).to(torch.bfloat16).view(torch.int16))
    assert bool(R.split_valid(hi, lo).all())
    # hi rounded toward zero instead of to nearest: hi + lo stays within ~2^-16 of x, but the pair is no split
    y = _rand(10000, seed=2)
    hi, lo = R.split(y)
    hi_trunc = (y.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)
    lo2 = (y - hi_trunc.float()).to(torch.bfloat16)
    wrong = hi_trunc.view(torch.int16) != hi.view(torch.int16)
    caught = ~R.split_valid(hi_trunc, lo2)[wrong]
    # all but the few whose lo rounds onto the exact tie
    assert wrong.sum() > 4000 and float(caught.double().mean()) > 0.99, (int(wrong.sum()), float(caught.double().mean()))


# ------------------------------------------------------------------------------------------------ trunk
@pytest.mark.parametrize("H,W,pad_t,pad_l,cout", [(9, 7, 0, 1, 5), (10, 12, 2, 0, 8), (1, 1, 1, 1, 3), (7, 11, 2, 2, 64)])
def test_stem_matches_conv2d(H, W, pad_t, pad_l, cout):
    x = _rand(2, 3, H, W, seed=3)
    w, b = _rand(cout, 3, 3, 3, seed=4), _rand(cout, seed=5)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    ref = F.silu(F.conv2d(F.pad(x.double(), (pad_l, 2 * Wo + 2, pad_t, 2 * Ho + 2)), w.double(), b.double(), stride=2))
    ref = ref[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    got = R.stem(x, w, b, Ho, Wo, pad_t, pad_l, 64)
    _close(got["y"][..., :cout], ref)
    assert not got["y"][..., cout:].any()
    assert bool((got["mag"][..., :cout] >= got["y"][..., :cout].abs() / 1.1 - 1e-12).all())


@pytest.mark.parametrize("k,s,pad_t,pad_l,C,cs,H,W", [(3, 1, 1, 1, 8, 64, 9, 13), (3, 2, 0, 2, 16, 128, 10, 7),
                                                      (5, 1, 4, 1, 24, 64, 6, 9), (5, 2, 3, 0, 8, 64, 11, 12),
                                                      (5, 2, 2, 2, 40, 64, 1, 5)])
def test_depthwise_matches_grouped_conv2d(k, s, pad_t, pad_l, C, cs, H, W):
    x = _rand(2, H, W, C, seed=6)
    hi, lo = _planes(x, cs, junk_seed=7)                 # channels [C, cs) must not be read
    w, b = _rand(k * k, C, seed=8), _rand(C, seed=9)
    Ho, Wo = max((H + pad_t - k) // s + 1, 1), max((W + pad_l - k) // s + 1, 1)
    xv = (hi.double() + lo.double())[..., :C].permute(0, 3, 1, 2)
    wk = w.double().t().reshape(C, 1, k, k)
    ref = F.conv2d(F.pad(xv, (pad_l, s * Wo + k, pad_t, s * Ho + k)), wk, b.double(), stride=s, groups=C)
    ref = F.silu(ref[:, :, :Ho, :Wo]).permute(0, 2, 3, 1)
    got = R.dw(hi, lo, w, b, k, s, pad_t, pad_l, Ho, Wo, C)
    _close(got["y"], ref)
    _close(got["sums"], ref.sum((1, 2)))
    mag = F.conv2d(F.pad(xv.abs(), (pad_l, s * Wo + k, pad_t, s * Ho + k)), wk.abs(), b.double().abs(), stride=s,
                   groups=C)[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    _close(got["mag"], mag)
    _close(got["sums_mag"], (mag + ref.abs()).sum((1, 2)))


def test_se_gate_and_weights():
    n, C, R_, cout = 3, 70, 5, 130
    sums = _rand(n, 80, seed=10, scale=50.0)
    sums[:, C:] = float("nan")                              # read through sums_stride: never past C
    w_r, b_r, w_e, b_e = _rand(R_, C, seed=11), _rand(R_, seed=12), _rand(C, R_, seed=13), _rand(C, seed=14)
    got = R.se_gate(sums, C, 1.0 / 49, w_r, b_r, w_e, b_e)
    m = sums[:, :C].double() * R.f32(1.0 / 49)
    ref = torch.sigmoid(F.silu(m @ w_r.double().t() + b_r.double()) @ w_e.double().t() + b_e.double())
    _close(got["gate"], ref)
    w_p = _rand(cout, C, seed=15)
    full = R.se_weights(w_p, got["gate"], C, cout)
    # pack by hand into [chunk][kb][plane][bn][64] and unpack with the reference
    chunks, total = R.se_layout(C, cout)
    kb = -(-C // 64)
    packed = torch.zeros(n, total, dtype=torch.float64)
    for n0, nn_, bn, off in chunks:
        blk = packed[:, off:off + kb * 2 * bn * 64].view(n, kb, 2, bn, 64)
        blk[:, :, 0] = full[:, n0:n0 + bn].reshape(n, bn, kb, 64).permute(0, 2, 1, 3)
    assert torch.equal(full[:, :cout, :C], w_p.double() * got["gate"].unsqueeze(1))
    assert not full[:, cout:].any() and not full[:, :, C:].any()
    hi, lo = R.se_unpack(packed, C, cout)
    assert torch.equal(hi, full)


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libstp3_b200.so is not built")
    return _lib.lib()


def test_se_layout_matches_the_library(L):
    for cout in range(1, 521):
        chunks, total = R.se_layout(96, cout)
        assert [(n0, n, bn) for n0, n, bn, _ in chunks] == dense.se_chunks(cout), cout
        for C in (8, 96, 4096):
            assert L.stp3_se_proj_weight_elems(C, cout) == R.se_layout(C, cout)[1], (C, cout)


# ------------------------------------------------------------------------------------------------ layout glue
@pytest.mark.parametrize("cl", [0, 1])
def test_layout_conversions(cl):
    n, C, H, W, cp = 2, 37, 3, 11, 64
    x = _rand(n, C, H, W, seed=16)
    src = x.permute(0, 2, 3, 1).contiguous() if cl else x
    hi, lo = R.f32_to_hilo(src, cl, n, C, H, W, cp)
    h2, l2 = dense.split_hilo(x.permute(0, 2, 3, 1))
    assert torch.equal(hi[..., :C], h2) and torch.equal(lo[..., :C], l2)
    assert not hi[..., C:].view(torch.int16).any() and not lo[..., C:].view(torch.int16).any()
    back = R.hilo_to_f32(hi, lo, n, H, W, cp, 5, 20)
    assert torch.equal(back, (h2.float() + l2.float()).permute(0, 3, 1, 2)[:, 5:25])
    s = R.spatial_sum(hi, lo, n, H * W, cp)
    _close(s["sums"], (hi.double() + lo.double()).sum((1, 2)).reshape(n, cp))


@pytest.mark.parametrize("mode", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cl", [0, 1])
def test_f32_to_plane_layouts(mode, cl):
    """both layouts land channels-last with +0 padding; the values are torch's rounding, -0.0 kept"""
    n, C, H, W, cp = 2, 37, 3, 11, 64
    x = _rand(n, C, H, W, seed=17) * 1e3
    x[0, 1, 2, 3] = -0.0
    src = x.permute(0, 2, 3, 1).contiguous() if cl else x
    p = R.f32_to_plane(src, cl, n, C, H, W, cp, mode)
    assert p.dtype == mode and p.shape == (n, H, W, cp)
    assert torch.equal(p[..., :C].view(torch.int16), x.permute(0, 2, 3, 1).to(mode).view(torch.int16))
    assert not p[..., C:].view(torch.int16).any()
    assert torch.signbit(p[0, 2, 3, 1].float())


# ------------------------------------------------------------------------------------------------ small dense layers
@pytest.mark.parametrize("temporal,n_const,accumulate,with_bias", [(True, 0, False, True), (True, 2, True, True),
                                                                   (False, 3, False, False), (True, 0, False, False)])
def test_pool_bias_matches_avg_pool3d(temporal, n_const, accumulate, with_bias):
    B, T, C, R_, CO, hw = 2, 3, 9, 4, 7, 20
    n = B * T
    sums = _rand(n, C + 3, seed=17, scale=10.0)
    const = _rand(n, n_const, seed=18) if n_const else None
    W1, b1, W2 = _rand(R_, C, seed=19), _rand(R_, seed=20), _rand(CO, R_, seed=21)
    bias = _rand(CO, seed=22) if with_bias else None
    prior = _rand(n, CO + 2, seed=23)
    got = R.pool_bias(sums, n, T, C, 1.0 / hw, temporal, const, n_const, W1, b1, W2, bias, prior, accumulate)
    m = sums[:, :C - n_const].double() * R.f32(1.0 / hw)
    if n_const:
        m = torch.cat([m, const.double()], 1)
    if temporal:   # AvgPool3d((2, 1, 1)), time padding 1, count_include_pad=False; frame t pools {t-1, t}
        m = F.avg_pool3d(m.view(B, T, C).permute(0, 2, 1)[..., None, None], (2, 1, 1), stride=1, padding=(1, 0, 0),
                         count_include_pad=False)[:, :, :T, 0, 0].permute(0, 2, 1).reshape(n, C)
    base = prior[:, :CO].double() if accumulate else bias.double().expand(n, CO) if with_bias else 0
    _close(got["out"], base + F.relu(m @ W1.double().t() + b1.double()) @ W2.double().t())


def test_small_linear_rules():
    x, W, bias, prior = _rand(4, 6, seed=24), _rand(5, 6, seed=25), _rand(5, seed=26), _rand(4, 9, seed=27)
    lin = x.double() @ W.double().t()
    _close(R.small_linear(x, W, bias, prior, True)["out"], prior[:, :5].double() + lin)
    _close(R.small_linear(x, W, bias, prior, False)["out"], bias.double() + lin)
    _close(R.small_linear(x, W, None, prior, False)["out"], lin)


@pytest.mark.parametrize("h,w,skip", [(5, 7, True), (1, 4, False), (3, 1, True), (1, 1, True)])
def test_upsample_matches_interpolate(h, w, skip):
    C, xcs, scs, s_coff = 8, 64, 64, 16
    x = _rand(2, h, w, C, seed=28)
    xh, xl = _planes(x, xcs, junk_seed=29)
    sh, sl = _planes(_rand(2, 2 * h, 2 * w, scs, seed=30), scs)
    got = R.upsample2x_add(xh, xl, 2, h, w, C, sh if skip else None, sl if skip else None, s_coff)
    xv = (xh.double() + xl.double())[..., :C].permute(0, 3, 1, 2)
    ref = F.interpolate(xv, scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    if skip:
        ref = ref + (sh.double() + sl.double())[..., s_coff:s_coff + C]
    _close(got["y"], ref)


# ------------------------------------------------------------------------------------------------ refusals
F1 = 1 << 20            # a non-null, 16-byte aligned pointer: never dereferenced, every call below is refused


def _refused(L, code, needle):
    assert code != 0
    msg = L.stp3_last_error().decode()
    assert needle in msg, msg


def test_refusals(L):
    stem = lambda **kw: L.stp3_effnet_stem(*dict(dict(x=F1, n=2, H=16, W=16, Ho=8, Wo=8, pt=0, pl=1, w=F1, b=F1,   # noqa: E731
                                                      cout=32, cs=64, hi=F1, lo=F1), **kw).values(), None)
    _refused(L, stem(w=None), "null pointer")
    _refused(L, stem(Ho=0), "non-positive")
    _refused(L, stem(cout=65, cs=128), "cout must be <= 64")
    _refused(L, stem(cs=96), "multiple of 64")
    _refused(L, stem(pt=3), "pad out of range")
    _refused(L, stem(hi=F1 + 8), "16-byte aligned")
    _refused(L, stem(lo=F1 + 2), "16-byte aligned")
    _refused(L, stem(n=32768, Ho=2048, Wo=2048), "2^31 - 1 blocks")        # 2^31 blocks, below the old 2^40 bound

    def desc(**kw):
        return _lib.DwDesc(**dict(dict(n_img=2, H=16, W=16, Ho=16, Wo=16, k=3, stride=1, pad_t=1, pad_l=1, C=64,
                                       in_cstride=64, out_cstride=64), **kw))

    def dw(sums=None, scratch=None, nbytes=0, hi=F1, **kw):       # every call below must be refused: F1 is no buffer
        return L.stp3_dw_fwd(ctypes.byref(desc(**kw)), hi, F1, F1, F1, F1, F1, sums, scratch, nbytes, None)
    _refused(L, dw(hi=None), "null pointer")
    _refused(L, dw(k=4), "k must be 3 or 5")
    _refused(L, dw(stride=3), "stride must be 1 or 2")
    _refused(L, dw(pad_t=3), "pad out of range")
    _refused(L, dw(C=12), "multiple of 8")
    _refused(L, dw(C=128), "multiple of 8")
    _refused(L, dw(hi=F1 + 8), "16-byte aligned")
    need = L.stp3_dw_sums_scratch_bytes(ctypes.byref(desc()))
    assert need == 2 * 2 * 64 * 4                         # 2 images x 2 tiles of 8 x 16 x C floats
    _refused(L, dw(sums=F1, scratch=F1, nbytes=need - 4), "scratch")
    _refused(L, dw(sums=F1, scratch=None, nbytes=need), "scratch")
    _refused(L, dw(n_img=65536), "too many images")

    se = lambda **kw: L.stp3_se_gate(*dict(dict(s=F1, ss=64, n=2, C=64, inv=0.1, wr=F1, br=F1, R=8, we=F1, be=F1,   # noqa: E731
                                                wp=F1, cout=32, g=F1, wi=F1), **kw).values(), None)
    _refused(L, se(wi=None), "null pointer")
    _refused(L, se(ss=63), "bad dimensions")
    _refused(L, se(C=4097, ss=4097), "C <= 4096")
    _refused(L, se(R=1025), "R <= 1024")

    _refused(L, L.stp3_f32_to_hilo(F1, 0, 2, 65, 4, 4, 64, F1, F1, None), "bad argument")
    _refused(L, L.stp3_f32_to_hilo(F1, 0, 65536, 8, 4, 4, 64, F1, F1, None), "65535 images")
    _refused(L, L.stp3_hilo_to_f32(F1, F1, 2, 4, 4, 64, 8, 57, F1, None), "bad argument")
    _refused(L, L.stp3_hilo_to_f32(F1, F1, 2, 0, 4, 64, 0, 8, F1, None), "non-positive H or W")
    _refused(L, L.stp3_hilo_to_f32(F1, F1, 2, 4, -1, 64, 0, 8, F1, None), "non-positive H or W")
    _refused(L, L.stp3_hilo_to_f32(F1, F1, 65536, 4, 4, 64, 0, 8, F1, None), "65535 images")
    _refused(L, L.stp3_spatial_sum(F1, F1, 2, 16, 1025, F1, None), "bad argument")
    _refused(L, L.stp3_spatial_sum(F1, F1, 65536, 16, 64, F1, None), "65535 images")

    pool = lambda **kw: L.stp3_pool_bias(*dict(dict(s=F1, ss=64, n=6, T=3, C=64, inv=0.1, tmp=1, cv=None, nc=0,   # noqa: E731
                                                    W1=F1, b1=F1, R=16, W2=F1, CO=64, bias=None, out=F1, cos=64,
                                                    acc=0), **kw).values(), None)
    _refused(L, pool(nc=64, cv=F1), "bad argument")
    _refused(L, pool(nc=2), "bad argument")                 # constants without their values
    _refused(L, pool(CO=65), "bad argument")
    _refused(L, pool(ss=32), "bad argument")
    _refused(L, pool(C=12000, R=289, ss=12000), "C + R must be <= 12288")
    _refused(L, L.stp3_small_linear(F1, F1, 4, 6, 65, None, F1, 64, 0, None), "bad argument")
    _refused(L, L.stp3_small_linear(F1, None, 4, 6, 6, None, F1, 64, 0, None), "bad argument")

    up = lambda **kw: L.stp3_upsample2x_add(*dict(dict(xh=F1, xl=F1, n=2, h=4, w=4, xcs=64, sh=F1, sl=F1, scs=64,   # noqa: E731
                                                       soff=0, yh=F1, yl=F1, ycs=64, yoff=0, C=64), **kw).values(), None)
    _refused(L, up(h=0), "null/empty")
    _refused(L, up(sl=None), "both skip planes")
    _refused(L, up(C=60), "multiples of 8")
    _refused(L, up(yoff=8), "multiples of 8")
    _refused(L, up(xh=F1 + 8), "16-byte aligned")
    _refused(L, up(sl=F1 + 2), "16-byte aligned")
    _refused(L, up(yl=F1 + 8), "16-byte aligned")


# ------------------------------------------------------------------------------------------------ recorder guard
# entry point -> the dense function that wraps it (tests/test_aux_contract_gpu.py records these functions)
WRAPPERS = {"stp3_effnet_stem": "effnet_stem", "stp3_dw_fwd": "dw_conv", "stp3_se_gate": "se_gate",
            "stp3_f32_to_hilo": "from_f32", "stp3_hilo_to_f32": "to_f32", "stp3_spatial_sum": "spatial_sum",
            "stp3_pool_bias": "pool_bias", "stp3_small_linear": "small_linear", "stp3_upsample2x_add": "upsample2x_add"}


def aux_calls_outside_the_wrappers():
    """Uses of the nine entry points and of stp3_f32_to_plane anywhere in the package except inside their dense.py
    wrapper (and stp3_f32_to_hilo / stp3_f32_to_plane inside dense_train.to_hl), and imports of a wrapper by name: each would launch a kernel the
    recorder does not see.  (A bare call inside the wrapper's own module resolves the module attribute the recorder
    replaces, so it is recorded.)"""
    pkg = os.path.dirname(os.path.abspath(dense.__file__))
    allowed = {(os.path.abspath(dense.__file__), fn, sym) for sym, fn in WRAPPERS.items()}
    allowed |= {(os.path.abspath(dense_train.__file__), "to_hl", sym) for sym in ("stp3_f32_to_hilo", "stp3_f32_to_plane")}
    symbols = set(WRAPPERS) | {"stp3_f32_to_plane"}
    wrappers = set(WRAPPERS.values())
    bad = []
    for root, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            path = os.path.join(root, f)
            with open(path) as fh:
                tree = ast.parse(fh.read())
            for top in ast.walk(tree):
                if isinstance(top, ast.ImportFrom) and any(a.name in wrappers | {"to_hl"} for a in top.names):
                    bad.append(f"{f}:{top.lineno} imports {[a.name for a in top.names]}")
            owner = {}
            for fn in ast.walk(tree):
                if isinstance(fn, (ast.FunctionDef, ast.AsyncFunctionDef)):
                    for n in ast.walk(fn):
                        owner.setdefault(id(n), fn.name)     # the outermost function wins (ast.walk is breadth first)
            for n in ast.walk(tree):
                if isinstance(n, ast.Attribute) and n.attr in symbols:
                    if (path, owner.get(id(n)), n.attr) not in allowed:
                        bad.append(f"{f}:{n.lineno} {n.attr} in {owner.get(id(n))}")
    return bad


def test_every_call_goes_through_a_recorded_wrapper():
    assert not aux_calls_outside_the_wrappers()
