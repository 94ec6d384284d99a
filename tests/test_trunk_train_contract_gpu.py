"""GPU: every launch of the trunk's train-mode entry points, recorded from real train steps of the b0 and b4 trunks and
replayed against an fp64 model of its contract (the pattern of tests/test_train_contract_gpu.py).

The recorder wraps the host calls of dense_train (stem_raw, stem_wgrad, dw_raw, dw_dgrad, dw_wgrad, bn_act, bn_act_grad,
image_channel_dot, se_backward) during the train steps of tests/test_train_contract_gpu.py trunk_step (b0 and b4 on
3 x 35 x 51 images, b4 on one frame of six 224 x 480 cameras), keeping copies of their operands and results.
Synthetic launches in the same argument forms add what no step makes: every partition of the three partitioned
reductions (one part, several, a ragged last part, the 256-part cap; tests/trunk_train_reference.py mirrors the
partition), the stem at cout 1 and 64 and with a one-pixel output, depthwise pad_t != pad_l and one-row or one-column
outputs, the channel dot over hundreds of images, stp3_se_bwd at its limits, swish saturated in both BatchNorm passes.
Each launch is replayed through the C entry point on sentinel-filled (NaN) outputs, with the depthwise operands inside
wider rows whose extra channels hold NaN (row strides > C), and must
  - write every element of its window and nothing outside it,
  - equal the production launch bit for bit (and itself on a second replay),
  - hold its fp64 model: elementwise kernels within a few fp32 ulps of the summed magnitudes, reductions within one
    rounding of the exact sum of their fp32 terms (plus the fp64 rounding of the partials).
stp3_trunk_bn_act is also replayed writing its planes only (no fp32 output).  The coverage test asserts that every entry
point and listed feature was reached, and a last test that a trunk step calls no library entry point that a suite
replaying the trunk steps does not check."""
import collections
import ctypes
import importlib
import time

import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import _lib, dense, dense_train as T
from tests import test_train_contract_gpu as TC
from tests import trunk_train_reference as TR

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ULP = 2.0 ** -24
NAMES = ("stem_raw", "stem_wgrad", "dw_raw", "dw_dgrad", "dw_wgrad", "bn_act", "bn_act_grad", "image_channel_dot",
         "se_backward")
SOURCES = tuple(TC.TRUNK_STEPS)


def _clone(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, T.BNStats):
        return T.BNStats(v.mean.clone(), v.var.clone(), v.invstd.clone(), v.n)
    if isinstance(v, dense.HL):
        return dense.HL(v.hi.clone(), v.lo.clone() if v.lo is not None else None, v.c)
    if isinstance(v, torch.nn.Module):
        return (v.weight.detach().clone(), v.bias.detach().clone())
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(u) for u in v)
    return v


_RECORDS = {}


def records(source):
    """every call of the NAMES entry points of dense_train during one trunk step (tests/test_train_contract_gpu.py
    trunk_step) -> [(name, args, kwargs, result)], all cloned"""
    if source in _RECORDS:
        return _RECORDS[source]
    rec = []
    originals = {n: getattr(T, n) for n in NAMES}

    def wrap(name, fn):
        def f(*a, **kw):
            out = fn(*a, **kw)
            rec.append((name, _clone(a), _clone(kw), _clone(out)))
            return out
        return f
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    for n, fn in originals.items():
        setattr(T, n, wrap(n, fn))
    try:
        TC.trunk_step(*TC.TRUNK_STEPS[source])
    finally:
        for n, fn in originals.items():
            setattr(T, n, fn)
    print(f"\n{source}: {len(rec)} launches recorded in {time.time() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated")
    _RECORDS[source] = rec
    return rec


def _launches(name):
    """(source, index, (name, args, kwargs, production result or None)) of every recorded and synthetic launch"""
    out = [(src, i, r) for src in SOURCES for i, r in enumerate(records(src)) if r[0] == name]
    return out + [("synthetic", i, r) for i, r in enumerate(synthetic()) if r[0] == name]


_CHECKED = {}


def checked(name, check_one):
    """check_one(args, kwargs, production result) -> features, over every launch of `name` once -> [(source, index,
    features)]"""
    if name not in _CHECKED:
        t0 = time.time()
        rows = []
        for src, i, (_, a, kw, out) in _launches(name):
            _CURRENT[:] = [name, src]
            key = (name, "synthetic" if src == "synthetic" else "recorded")
            WORST[key] = (WORST.get(key, (0.0, 0))[0], WORST.get(key, (0.0, 0))[1] + 1)
            rows.append((src, i, check_one(a, kw, out)))
        print(f"\n{name}: {len(rows)} launches checked in {time.time() - t0:.1f} s")
        _CHECKED[name] = rows
    return _CHECKED[name]


def _same(reps, out):
    """two replays bitwise equal, and equal to the production result when there is one"""
    return torch.equal(reps[0], reps[1]) and (out is None or torch.equal(reps[0].contiguous(), out))


def ptr(t):
    return t.data_ptr() if t is not None else None


def stream():
    return torch.cuda.current_stream().cuda_stream


def wide(t, extra, fill=float("nan")):
    """t (..., C) inside rows of C + extra channels whose extra channels hold `fill`"""
    out = torch.full((*t.shape[:-1], t.shape[-1] + extra), fill, dtype=t.dtype, device=t.device)
    out[..., :t.shape[-1]] = t
    return out


def check_window(out, C, extra):
    assert torch.isnan(out[..., C:]).all(), "a launch wrote outside its window"
    assert not torch.isnan(out[..., :C]).any(), "a launch left part of its window unwritten (or read a NaN pad)"


# worst error of each entry point as a fraction of its bar: {(entry point, "recorded" / "synthetic"): (worst, launches)}
WORST = {}
_CURRENT = []          # (entry point, source) of the launch being checked


def _note(ratio):
    name, src = _CURRENT
    key = (name, "synthetic" if src == "synthetic" else "recorded")
    w, n = WORST.get(key, (0.0, 0))
    WORST[key] = (max(w, ratio), n)


def elementwise_ok(got, ref, mag, ulps):
    err = (got.double().cpu() - ref).abs()
    bar = ulps * ULP * mag + 1e-30
    _note(float((err / bar).max()))
    assert (err <= bar).all(), float((err / (mag + 1e-30)).max() / ULP)


def reduction_ok(got, exact, mag):
    err = (got.double().cpu() - exact).abs()
    bar = ULP * exact.abs() + 1e-13 * mag + 1e-37
    _note(float((err / bar).max()))
    assert (err <= bar).all(), float((err / bar).max())


# ------------------------------------------------------------------------------------------------ depthwise
def _pads(pad):
    return pad if isinstance(pad, tuple) else (pad, pad)


def dw_model(x, w, stride, pad, Ho, Wo):
    """x (N, H, W, C), w (C, 1, k, k), pad (top, left): zero padding, then the rows and columns the outputs read"""
    N, H, W, C = x.shape
    k = w.shape[-1]
    pt, pl = pad
    pb, pr = (Ho - 1) * stride + k - H - pt, (Wo - 1) * stride + k - W - pl
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb)), w, stride=stride, groups=C).permute(0, 2, 3, 1)


def _desc(N, H, W, Ho, Wo, k, s, pad, C, ics, ocs):
    pt, pl = pad
    return _lib.DwDesc(n_img=N, H=H, W=W, Ho=Ho, Wo=Wo, k=k, stride=s, pad_t=pt, pad_l=pl, C=C, in_cstride=ics,
                       out_cstride=ocs)


def _dw_check(name):
    def one(a, kw, out):
        L = _lib.lib()
        if name == "dw_raw":
            x, w, s, pad, (Ho, Wo) = a
            N, H, W, C = x.shape
        elif name == "dw_dgrad":
            g, w, s, pad, (H, W) = a
            N, Ho, Wo, C = g.shape
        else:
            x, g, k, s, pad = a
            N, H, W, C = x.shape
            Ho, Wo = g.shape[1:3]
        k = a[1].shape[-1] if name != "dw_wgrad" else a[2]
        pad = _pads(pad)
        f = {name, f"dw k{k} s{s}"}
        if C % 32:
            f.add("dw C % 32 != 0, wide rows")
        if pad[0] != pad[1]:
            f.add("dw pad_t != pad_l")
        if Ho == 1 or Wo == 1:
            f.add("dw Ho or Wo 1")
        ei, eo = 5, 3                  # every replay reads and writes rows wider than C, the extra channels NaN
        d = _desc(N, H, W, Ho, Wo, k, s, pad, C, C + ei, C + eo)
        reps = []
        for _ in range(2):
            if name == "dw_raw":
                xw = wide(x, ei)
                y = torch.full((N, Ho, Wo, C + eo), float("nan"), device=DEV)
                wt = T._dw_taps(w)
                assert L.stp3_dw_fwd_raw(ctypes.byref(d), ptr(xw), ptr(wt), ptr(y), stream()) == 0
                check_window(y, C, eo)
                reps.append(y[..., :C])
            elif name == "dw_dgrad":
                gw = wide(g, eo)
                dx = torch.full((N, H, W, C + ei), float("nan"), device=DEV)
                wt = T._dw_taps(w)
                assert L.stp3_dw_dgrad(ctypes.byref(d), ptr(gw), ptr(wt), ptr(dx), stream()) == 0
                check_window(dx, C, ei)
                reps.append(dx[..., :C])
            else:
                xw, gw = wide(x, ei), wide(g, eo)
                nbytes = L.stp3_dw_wgrad_scratch_bytes(ctypes.byref(d))
                scratch = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
                dw = torch.full((k * k, C), float("nan"), device=DEV)
                assert L.stp3_dw_wgrad(ctypes.byref(d), ptr(xw), ptr(gw), ptr(dw), ptr(scratch), nbytes,
                                       stream()) == 0
                assert not torch.isnan(dw).any()
                reps.append(dw.t().reshape(C, 1, k, k))
                parts = TR.dw_wgrad_parts(N, Ho, Wo)
                assert nbytes == parts * k * k * C * 8
                f |= TR.part_features("dw", N * Ho * Wo, parts, 512)
        torch.cuda.synchronize()
        assert _same(reps, out), (name, tuple(x.shape if name != "dw_dgrad" else g.shape))
        got = reps[0]
        if name == "dw_raw":
            x64, w64 = x.double().cpu(), w.double().cpu()
            elementwise_ok(got, dw_model(x64, w64, s, pad, Ho, Wo), dw_model(x64.abs(), w64.abs(), s, pad, Ho, Wo),
                           2 * k * k)
        elif name == "dw_dgrad":
            w64 = w.double().cpu()
            x0 = torch.zeros(N, H, W, C, dtype=torch.float64, requires_grad=True)
            exact, = torch.autograd.grad(dw_model(x0, w64, s, pad, Ho, Wo), [x0], g.double().cpu())
            x1 = torch.zeros(N, H, W, C, dtype=torch.float64, requires_grad=True)
            mag, = torch.autograd.grad(dw_model(x1, w64.abs(), s, pad, Ho, Wo), [x1], g.double().cpu().abs())
            elementwise_ok(got, exact, mag, 2 * k * k)
        else:
            wr = torch.zeros(C, 1, k, k, dtype=torch.float64, requires_grad=True)
            exact, = torch.autograd.grad(dw_model(x.double().cpu(), wr, s, pad, Ho, Wo), [wr], g.double().cpu())
            wr = torch.zeros(C, 1, k, k, dtype=torch.float64, requires_grad=True)
            mag, = torch.autograd.grad(dw_model(x.double().cpu().abs(), wr, s, pad, Ho, Wo), [wr],
                                       g.double().cpu().abs())
            reduction_ok(got, exact, mag)
        return f
    return one


def test_depthwise_launches():
    for name in ("dw_raw", "dw_dgrad", "dw_wgrad"):
        checked(name, _dw_check(name))


# ------------------------------------------------------------------------------------------------ stem
def stem_model(x, w, pad, Ho, Wo):
    H, W = x.shape[2:]
    pt, pl = pad
    pb, pr = (Ho - 1) * 2 + 3 - H - pt, (Wo - 1) * 2 + 3 - W - pl
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, stride=2).permute(0, 2, 3, 1)


def _stem_features(cout, Ho, Wo):
    return {f"stem cout {cout}"} | ({"stem one-pixel output"} if Ho == Wo == 1 else set())


def _stem_raw_check(a, kw, out):
    L = _lib.lib()
    x, w, (Ho, Wo), pad = a
    pad = _pads(pad)
    M, _, H, W = x.shape
    cout = w.shape[0]
    reps = []
    for _ in range(2):
        y = torch.full((M, Ho, Wo, cout), float("nan"), device=DEV)
        assert L.stp3_effnet_stem_raw(ptr(x), M, H, W, Ho, Wo, *pad, ptr(w.contiguous()), cout, ptr(y),
                                      stream()) == 0
        reps.append(y)
    torch.cuda.synchronize()
    assert _same(reps, out)
    x64, w64 = x.double().cpu(), w.double().cpu()
    elementwise_ok(reps[0], stem_model(x64, w64, pad, Ho, Wo), stem_model(x64.abs(), w64.abs(), pad, Ho, Wo), 60)
    return {"stem_raw"} | _stem_features(cout, Ho, Wo)


def _stem_wgrad_check(a, kw, out):
    L = _lib.lib()
    x, g, pad = a
    pad = _pads(pad)
    M, _, H, W = x.shape
    _, Ho, Wo, cout = g.shape
    nbytes = L.stp3_effnet_stem_wgrad_scratch_bytes(M, Ho, Wo, cout)
    parts = TR.stem_wgrad_parts(M, Ho, Wo)
    assert nbytes == parts * cout * 27 * 8
    reps = []
    for _ in range(2):
        dw = torch.full((cout, 3, 3, 3), float("nan"), device=DEV)
        scratch = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
        assert L.stp3_effnet_stem_wgrad(ptr(x), M, H, W, Ho, Wo, *pad, ptr(g), cout, ptr(dw), ptr(scratch),
                                        nbytes, stream()) == 0
        reps.append(dw)
    torch.cuda.synchronize()
    assert _same(reps, out)
    wr = torch.zeros(cout, 3, 3, 3, dtype=torch.float64, requires_grad=True)
    exact, = torch.autograd.grad(stem_model(x.double().cpu(), wr, pad, Ho, Wo), [wr], g.double().cpu())
    wr = torch.zeros(cout, 3, 3, 3, dtype=torch.float64, requires_grad=True)
    mag, = torch.autograd.grad(stem_model(x.double().cpu().abs(), wr, pad, Ho, Wo), [wr], g.double().cpu().abs())
    reduction_ok(reps[0], exact, mag)
    return {"stem_wgrad"} | _stem_features(cout, Ho, Wo) | TR.part_features("stem", M * Ho * Wo, parts, 1024)


def test_stem_launches():
    checked("stem_raw", _stem_raw_check)
    checked("stem_wgrad", _stem_wgrad_check)


# ------------------------------------------------------------------------------------------------ BatchNorm passes
def _vectors(st, gb):
    if st is None:
        return None, None, None, None
    return st.mean, st.invstd, gb[0].float().contiguous(), gb[1].float().contiguous()


def _z64(x, st, gb):
    if st is None:
        return x.double().cpu(), x.double().cpu().abs()
    m, i, g, b = (t.double().cpu() for t in _vectors(st, gb))
    z = (x.double().cpu() - m) * i * g + b
    mag = (x.double().cpu().abs() + m.abs()) * i * g.abs() + b.abs()
    return z, mag


def _bn_act_check(a, kw, out):
    L = _lib.lib()
    x, st, gb = a[:3]
    swish = a[3] if len(a) > 3 else kw["swish"]
    mul, scale, res, hl = kw.get("mul"), kw.get("scale"), kw.get("res"), kw.get("hl", False)
    f = {"bn_act" + (" swish" if swish else "") + (" stats" if st is not None else "") +
         (" mul" if mul is not None else "") + (" scale" if scale is not None else "") +
         (" res" if res is not None else "") + (" planes" if hl else "")}
    N, H, W, C = x.shape
    mean, invstd, gam, bet = _vectors(st, gb)
    cp = dense.pad_to(C)
    runs = []
    for f32 in (True, True, False):             # twice with the fp32 output, once with the planes only
        y = torch.full_like(x, float("nan")) if f32 else None
        hi = torch.full((N, H, W, cp), float("nan"), dtype=torch.bfloat16, device=DEV)
        lo = torch.full_like(hi, float("nan"))
        assert L.stp3_trunk_bn_act(ptr(x), N * H * W, C, H * W, ptr(mean), ptr(invstd), ptr(gam), ptr(bet),
                                   int(swish), ptr(mul), ptr(scale), ptr(res), ptr(y), ptr(hi), ptr(lo), cp,
                                   stream()) == 0
        runs.append((y, hi, lo))
    torch.cuda.synchronize()
    (y0, h0, l0), (y1, h1, l1), (_, h2, l2) = runs
    assert torch.equal(y0, y1) and (out is None or torch.equal(y0, out[0]))
    assert torch.equal(h0, h1) and torch.equal(h0, h2) and torch.equal(l0, l2)
    assert (h0[..., C:] == 0).all() and (l0[..., C:] == 0).all()
    h2_, l2_ = dense.split_hilo(y0)
    assert torch.equal(h0[..., :C], h2_) and torch.equal(l0[..., :C], l2_), "the planes are not the split of y"
    if hl and out is not None:
        assert torch.equal(h0, out[1].hi.view_as(h0)) and torch.equal(l0, out[1].lo.view_as(l0))
    f.add("bn_act planes only")
    if cp > C:
        f.add("bn_act planes only, hl_cstride > C")
    z, mag = _z64(x, st, gb)
    if swish:                                  # |swish'| <= 1.1
        if bool((z.abs() >= 90).any()):
            f.add("bn_act swish saturated")
        sg = torch.sigmoid(z)
        z, mag = z * sg, 1.1 * mag + (z * sg).abs()
    n = N
    if mul is not None:
        mv = mul.double().cpu().view(n, 1, 1, C)
        z, mag = z * mv, mag * mv.abs()
    if scale is not None:
        sv = scale.double().cpu().view(n, 1, 1, 1)
        z, mag = z * sv, mag * sv.abs()
    if res is not None:
        z, mag = z + res.double().cpu(), mag + res.double().cpu().abs()
    elementwise_ok(y0, z, mag, 16)
    return f


def test_bn_act_launches():
    checked("bn_act", _bn_act_check)


def _bn_act_grad_check(a, kw, out):
    L = _lib.lib()
    g, x, st, gb = a[:4]
    swish = a[4] if len(a) > 4 else kw["swish"]
    mul, add, scale = kw.get("mul"), kw.get("add"), kw.get("scale")
    f = {"bn_act_grad" + (" swish" if swish else "") + (" mul" if mul is not None else "") +
         (" add" if add is not None else "") + (" scale" if scale is not None else "")}
    N, H, W, C = g.shape
    mean, invstd, gam, bet = _vectors(st, gb)
    reps = []
    for _ in range(2):
        o = torch.full_like(g, float("nan"))
        assert L.stp3_trunk_bn_act_bwd(ptr(g), ptr(x), N * H * W, C, H * W, ptr(mean), ptr(invstd), ptr(gam),
                                       ptr(bet), int(swish), ptr(mul), ptr(add), ptr(scale), ptr(o),
                                       stream()) == 0
        reps.append(o)
    torch.cuda.synchronize()
    assert _same(reps, out)
    r, mag = g.double().cpu(), g.double().cpu().abs()
    if mul is not None:
        mv = mul.double().cpu().view(N, 1, 1, C)
        r, mag = r * mv, mag * mv.abs()
    if add is not None:
        av = add.double().cpu().view(N, 1, 1, C)
        r, mag = r + av, mag + av.abs()
    if swish:
        z, _ = _z64(x, st, gb)
        if bool((z.abs() >= 90).any()):
            f.add("bn_act_grad swish saturated")
        sg = torch.sigmoid(z)
        d = sg * (1 + z * (1 - sg))
        # swish' is recomputed from z in fp32, and z carries a few ulps of its terms' magnitudes zm: that error enters
        # through |d swish'/dz| = s (1 - s) |2 + z (1 - 2 s)|, which in the saturated tail is |z| times swish' itself
        _, zm = _z64(x, st, gb)
        dd = sg * (1 - sg) * (2 + z.abs() * (1 - 2 * sg).abs()) * zm
        r, mag = r * d, mag * (sg * (1 + z.abs() * (1 - sg)) + dd)
    if scale is not None:
        sv = scale.double().cpu().view(N, 1, 1, 1)
        r, mag = r * sv, mag * sv.abs()
    # the recomputed z carries a few ulps of x's normalisation into swish'
    elementwise_ok(reps[0], r, mag, 64)
    return f


def test_bn_act_grad_launches():
    checked("bn_act_grad", _bn_act_grad_check)


# ------------------------------------------------------------------------------------------------ squeeze-excite
def _dot_check(a, kw, out):
    L = _lib.lib()
    y, u = a
    N, H, W, C = y.shape
    nbytes = L.stp3_image_channel_dot_scratch_bytes(N, H * W, C)
    parts = TR.dot_parts(H * W)
    assert nbytes == N * parts * C * 8
    reps = []
    for _ in range(2):
        o = torch.full((N, C), float("nan"), device=DEV)
        scratch = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
        assert L.stp3_image_channel_dot(ptr(y), ptr(u), N, H * W, C, ptr(o), ptr(scratch), nbytes, stream()) == 0
        reps.append(o)
    torch.cuda.synchronize()
    assert _same(reps, out)
    p = y.double().cpu() * u.double().cpu()
    reduction_ok(reps[0], p.sum(dim=(1, 2)), p.abs().sum(dim=(1, 2)))
    return {"image_channel_dot"} | TR.part_features("dot", H * W, parts, 256) | \
        ({"dot many images"} if N > 256 else set())


def test_image_channel_dot_launches():
    checked("image_channel_dot", _dot_check)


def _se_check(a, kw, out):
    L = _lib.lib()
    dgate, gate, sums, hw, w_r, b_r, w_e = a
    N, C = gate.shape
    R = w_r.shape[0]
    reps = []
    for _ in range(2):
        o = [torch.full((N, n), float("nan"), device=DEV) for n in (C, R, R, C)]
        assert L.stp3_se_bwd(ptr(dgate), ptr(gate), ptr(sums), N, C, 1.0 / hw, ptr(w_r), ptr(b_r), R, ptr(w_e),
                             *[ptr(t) for t in o], stream()) == 0
        reps.append(o)
    torch.cuda.synchronize()
    assert all(torch.equal(p, q) for p, q in zip(reps[0], reps[1]))
    assert out is None or all(torch.equal(p, r) for p, r in zip(reps[0], out))
    de, sr, dr, dmean = (t.double().cpu() for t in reps[0])
    g64, dg = gate.double().cpu(), dgate.double().cpu()
    m = sums.double().cpu() / hw
    Wr, br, We = w_r.double().cpu(), b_r.double().cpu(), w_e.double().cpu()
    r = m @ Wr.t() + br
    s = torch.sigmoid(r)
    de64 = dg * g64 * (1 - g64)
    dr64 = (de64 @ We) * s * (1 + r * (1 - s))
    # short fp32 dot products (length C or R) chained through swish': within 1e-5 of each output's max
    for got, ref in ((de, de64), (sr, r * s), (dr, dr64), (dmean, dr64 @ Wr / hw)):
        e = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        _note(e / 1e-5)
        assert e < 1e-5
    return {"se_backward", f"se_backward R {R}", f"se_backward C {C}"}


def test_se_backward_launches():
    checked("se_backward", _se_check)


# ------------------------------------------------------------------------------------------------ synthetic launches
def _rnd(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


_SYNTH = []


def synthetic():
    """Launches in the dense_train argument forms that no trunk step makes: every partition of the three partitioned
    reductions (one part, several, a ragged last part, the part cap), the stem at cout 1 and 64 and with a one-pixel
    output, depthwise rows of C % 32 != 0 channels, pad_t != pad_l, one-row and one-column outputs, the channel dot
    over many images, stp3_se_bwd at its limits (R = 1, R = 1024, C = 4096), swish saturated (|z| >= 90, where expf
    overflows) in both BatchNorm passes, and the gradient pass with mul, add, scale and swish at once."""
    if _SYNTH:
        return _SYNTH
    out = []
    # stem: (M, H, W, cout, pad); the first covers the part cap (282 204 > 256 * 1024 pixels) and a ragged last part
    for i, (M, H, W, cout, pad) in enumerate([(2, 701, 803, 1, (1, 1)), (1, 9, 9, 64, (0, 1)), (2, 2, 2, 8, (0, 0)),
                                              (1, 67, 129, 64, (1, 0))]):
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        x, w = _rnd(M, 3, H, W, seed=10 + i), _rnd(cout, 3, 3, 3, seed=20 + i, scale=0.3)
        g = _rnd(M, Ho, Wo, cout, seed=30 + i)
        out.append(("stem_raw", (x, w, (Ho, Wo), pad), {}, None))
        out.append(("stem_wgrad", (x, g, pad), {}, None))
    # depthwise: (N, H, W, C, k, s, pad); the first covers the cap and a ragged last part (160 801 pixels)
    for i, (N, H, W, C, k, s, pad) in enumerate([(1, 401, 401, 40, 3, 1, (1, 1)), (2, 17, 23, 24, 5, 2, (2, 1)),
                                                 (3, 2, 40, 70, 3, 2, (0, 1)), (2, 30, 1, 24, 5, 1, (2, 2)),
                                                 (1, 41, 31, 70, 3, 1, (1, 1)), (2, 33, 47, 56, 5, 2, (1, 2))]):
        Ho, Wo = (H + s - 1) // s, (W + s - 1) // s
        x, w = _rnd(N, H, W, C, seed=40 + i), _rnd(C, 1, k, k, seed=50 + i, scale=1.0 / k)
        g = _rnd(N, Ho, Wo, C, seed=60 + i)
        out.append(("dw_raw", (x, w, s, pad, (Ho, Wo)), {}, None))
        out.append(("dw_dgrad", (g, w, s, pad, (H, W)), {}, None))
        out.append(("dw_wgrad", (x, g, k, s, pad), {}, None))
    # image_channel_dot: (N, H, W, C): many images of one part, the cap with a ragged last part, several ragged parts
    for i, (N, H, W, C) in enumerate([(700, 3, 5, 70), (2, 300, 250, 40), (3, 7, 143, 33)]):
        out.append(("image_channel_dot", (_rnd(N, H, W, C, seed=70 + i), _rnd(N, H, W, C, seed=80 + i)), {}, None))
    # se_backward at the entry's limits
    for i, (N, C, R) in enumerate([(3, 16, 1), (2, 64, 1024), (2, 4096, 16)]):
        hw = 49
        gate = torch.sigmoid(_rnd(N, C, seed=90 + i, scale=2.0))
        out.append(("se_backward", (_rnd(N, C, seed=100 + i), gate, _rnd(N, C, seed=110 + i, scale=0.5 * hw), hw,
                                    _rnd(R, C, seed=120 + i, scale=C ** -0.5), _rnd(R, seed=130 + i, scale=0.1),
                                    _rnd(C, R, seed=140 + i, scale=R ** -0.5)), {}, None))
    # BatchNorm passes: z spread over +-300 (swish saturates where |z| >= 90), and every term of the gradient pass
    N, H, W, C = 3, 9, 13, 40
    x = _rnd(N, H, W, C, seed=150, scale=100.0)
    st = T.BNStats(_rnd(C, seed=151), _rnd(C, seed=152).abs() + 1.0, _rnd(C, seed=153).abs() + 0.5, N * H * W)
    gb = (_rnd(C, seed=154) + 1.5, _rnd(C, seed=155, scale=3.0))
    mul, add, scale = torch.sigmoid(_rnd(N, C, seed=156)), _rnd(N, C, seed=157), torch.tensor([0.0, 1.25, 1.25], device=DEV)
    out.append(("bn_act", (x, st, gb, True), {}, None))
    out.append(("bn_act", (x, st, gb, True), dict(mul=mul, scale=scale, res=_rnd(N, H, W, C, seed=158), hl=True), None))
    g = _rnd(N, H, W, C, seed=159)
    out.append(("bn_act_grad", (g, x, st, gb, True), dict(mul=mul, add=add, scale=scale), None))
    out.append(("bn_act_grad", (g, x / 100.0, st, gb, True), dict(mul=mul, add=add, scale=scale), None))
    _SYNTH.extend(out)
    return _SYNTH


# ------------------------------------------------------------------------------------------------ coverage
_CHECKS = {"dw_raw": _dw_check("dw_raw"), "dw_dgrad": _dw_check("dw_dgrad"), "dw_wgrad": _dw_check("dw_wgrad"),
           "stem_raw": _stem_raw_check, "stem_wgrad": _stem_wgrad_check, "bn_act": _bn_act_check,
           "bn_act_grad": _bn_act_grad_check, "image_channel_dot": _dot_check, "se_backward": _se_check}

REQUIRED = (["stem_raw", "stem_wgrad", "dw_raw", "dw_dgrad", "dw_wgrad", "image_channel_dot", "se_backward",
             "dw k3 s1", "dw k3 s2", "dw k5 s1", "dw k5 s2",
             "bn_act swish stats",                        # _bn0 / _bn1 / stem
             "bn_act mul planes",                         # the gate
             "bn_act stats scale res planes",             # _bn2 with drop-connect and skip, feeding an expand
             "bn_act stats planes",                       # _bn2 without skip
             "bn_act stats scale res",                    # the last block's _bn2
             "bn_act planes only", "bn_act planes only, hl_cstride > C", "bn_act swish saturated",
             "bn_act_grad swish", "bn_act_grad swish mul add", "bn_act_grad scale", "bn_act_grad swish mul add scale",
             "bn_act_grad swish saturated"]
            + [f"{k} {p}" for k in ("stem", "dw", "dot")
               for p in ("one part", "several parts", "ragged last part", "part cap")]
            + ["stem cout 1", "stem cout 64", "stem one-pixel output", "dw C % 32 != 0, wide rows", "dw pad_t != pad_l",
               "dw Ho or Wo 1", "dot many images", "se_backward R 1", "se_backward R 1024", "se_backward C 4096"])


def test_every_entry_point_and_path_was_reached():
    for src in SOURCES:
        assert {r[0] for r in records(src)} == set(NAMES), src
    counts = {f: 0 for f in REQUIRED}
    recorded = {f: 0 for f in REQUIRED}
    for name in NAMES:
        for src, _, feats in checked(name, _CHECKS[name]):
            for f in feats & set(REQUIRED):
                counts[f] += 1
                recorded[f] += src != "synthetic"
    print("\nfeature: launches (recorded from a trunk step)")
    for f in REQUIRED:
        print(f"  {f:<36s} {counts[f]:4d} ({recorded[f]})")
    print("worst error per entry point, as a fraction of its bar: recorded launches (trunk steps) / synthetic")
    for name in NAMES:
        (wr, nr), (ws, ns) = WORST.get((name, "recorded"), (0.0, 0)), WORST.get((name, "synthetic"), (0.0, 0))
        print(f"  {name:<18s} {wr:6.3f} over {nr:4d} / {ws:6.3f} over {ns:3d}")
    assert all(counts.values()), [f for f, c in counts.items() if not c]
    # at 224 x 480 the depthwise weight gradient reaches its part cap and ragged last parts in a real step
    big = [feats for name in ("dw_wgrad", "stem_wgrad") for src, _, feats in checked(name, _CHECKS[name])
           if src == "trunk_b4_224x480"]
    assert any("dw part cap" in f for f in big) and any("dw ragged last part" in f for f in big)


# ------------------------------------------------------------------------------------------------ no launch escapes
# Every entry point a trunk train step may call, and the suite that replays it from the trunk steps
SUITE_OF = {
    "stp3_conv_fwd": "test_conv_contract_gpu",
    **{e: "test_train_contract_gpu" for e in (
        "stp3_conv_wgrad", "stp3_conv_wgrad_scratch_bytes", "stp3_bn_stats", "stp3_bn_scratch_bytes",
        "stp3_bn_bwd_reduce", "stp3_bn_bwd_apply", "stp3_image_channel_sums", "stp3_image_channel_sums_scratch_bytes")},
    **{e: "test_aux_contract_gpu" for e in ("stp3_f32_to_hilo", "stp3_se_gate", "stp3_se_proj_weight_elems")},
    **{e: "test_trunk_train_contract_gpu" for e in (
        "stp3_effnet_stem_raw", "stp3_effnet_stem_wgrad", "stp3_effnet_stem_wgrad_scratch_bytes", "stp3_dw_fwd_raw",
        "stp3_dw_dgrad", "stp3_dw_wgrad", "stp3_dw_wgrad_scratch_bytes", "stp3_trunk_bn_act", "stp3_trunk_bn_act_bwd",
        "stp3_image_channel_dot", "stp3_image_channel_dot_scratch_bytes", "stp3_se_bwd")},
}


class _CountingLib:
    """stands in for the loaded library: counts every stp3_* entry point looked up (each lookup is one call)"""
    def __init__(self, lib):
        self._lib, self.calls = lib, collections.Counter()

    def __getattr__(self, name):
        if name.startswith("stp3_"):
            self.calls[name] += 1
        return getattr(self._lib, name)


def test_every_entry_point_of_a_trunk_step_is_replayed_by_a_suite(monkeypatch):
    counting = _CountingLib(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: counting)
    TC.trunk_step("b0", 3, 35, 51)
    monkeypatch.undo()
    print("\nentry points of a b0 train step at 3 x 35 x 51: calls (suite)")
    for e, n in sorted(counting.calls.items()):
        print(f"  {e:<40s} {n:5d}  ({SUITE_OF.get(e, 'NONE')})")
    unmapped = sorted(set(counting.calls) - set(SUITE_OF))
    assert not unmapped, f"entry points of a trunk step that no suite replays from the trunk steps: {unmapped}"
    assert {"stp3_conv_fwd", "stp3_conv_wgrad", "stp3_se_gate", "stp3_dw_wgrad"} <= set(counting.calls)
    for suite in sorted({SUITE_OF[e] for e in counting.calls}):
        mod = importlib.import_module(f"tests.{suite}")
        assert any(k.endswith(n) for k in mod.SOURCES for n in TC.TRUNK_STEPS), f"{suite} records no trunk step"
