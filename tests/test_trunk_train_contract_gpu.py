"""GPU: every launch of the trunk's train-mode entry points, recorded from real train steps of the b0 and b4 trunks and
replayed against an fp64 model of its contract (the pattern of tests/test_train_contract_gpu.py).

The recorder wraps the host calls of dense_train (stem_raw, stem_wgrad, dw_raw, dw_dgrad, dw_wgrad, bn_act, bn_act_grad,
image_channel_dot, se_backward) during a forward and backward, keeping copies of their operands and results.  Each
launch is then replayed through the C entry point on sentinel-filled (NaN) outputs, with the depthwise operands inside
wider rows whose extra channels hold NaN (row strides > C), and must
  - write every element of its window and nothing outside it,
  - equal the production launch bit for bit (and itself on a second replay),
  - hold its fp64 model: elementwise kernels within a few fp32 ulps of the summed magnitudes, reductions within one
    rounding of the exact sum of their fp32 terms (plus the fp64 rounding of the partials).
stp3_trunk_bn_act is also replayed writing its planes only (no fp32 output).  A last test asserts that every entry point
and path was reached."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet_oracle as EO
from stp3_b200 import _lib, dense, dense_train as T
from stp3_b200.models import efficientnet as EN

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ULP = 2.0 ** -24
NAMES = ("stem_raw", "stem_wgrad", "dw_raw", "dw_dgrad", "dw_wgrad", "bn_act", "bn_act_grad", "image_channel_dot",
         "se_backward")
REACHED = set()


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


def records(version):
    if version in _RECORDS:
        return _RECORDS[version]
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=3), version)
    nat = EN.EfficientNetTrunk(version, trainable=True)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to(DEV).train()
    rec = []
    originals = {n: getattr(T, n) for n in NAMES}

    def wrap(name, fn):
        def f(*a, **kw):
            out = fn(*a, **kw)
            rec.append((name, _clone(a), _clone(kw), _clone(out)))
            return out
        return f
    for n, fn in originals.items():
        setattr(T, n, wrap(n, fn))
    try:
        torch.manual_seed(5)
        x = torch.randn(3, 3, 35, 51, generator=torch.Generator().manual_seed(1)).to(DEV)
        r3, r4 = nat(x)
        (r3.square().sum() + r4.sum()).backward()
        torch.cuda.synchronize()
    finally:
        for n, fn in originals.items():
            setattr(T, n, fn)
    _RECORDS[version] = rec
    return rec


def _launches(name):
    return [(v, i, r) for v in ("b0", "b4") for i, r in enumerate(records(v)) if r[0] == name]


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


def elementwise_ok(got, ref, mag, ulps):
    err = (got.double().cpu() - ref).abs()
    assert (err <= ulps * ULP * mag + 1e-30).all(), float((err / (mag + 1e-30)).max() / ULP)


def reduction_ok(got, exact, mag):
    err = (got.double().cpu() - exact).abs()
    assert (err <= ULP * exact.abs() + 1e-13 * mag + 1e-37).all()


# ------------------------------------------------------------------------------------------------ depthwise
def dw_model(x, w, stride, pad, Ho, Wo):
    N, H, W, C = x.shape
    k = w.shape[-1]
    pb, pr = (Ho - 1) * stride + k - H - pad, (Wo - 1) * stride + k - W - pad
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (pad, pr, pad, pb)), w, stride=stride, groups=C).permute(0, 2, 3, 1)


def _desc(N, H, W, Ho, Wo, k, s, pad, C, ics, ocs):
    return _lib.DwDesc(n_img=N, H=H, W=W, Ho=Ho, Wo=Wo, k=k, stride=s, pad_t=pad, pad_l=pad, C=C, in_cstride=ics,
                       out_cstride=ocs)


def test_depthwise_launches():
    L = _lib.lib()
    for name in ("dw_raw", "dw_dgrad", "dw_wgrad"):
        for v, i, (_, a, kw, out) in _launches(name):
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
            REACHED.add(f"dw k{k} s{s}")
            ei, eo = 5, 3
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
            torch.cuda.synchronize()
            assert torch.equal(reps[0], reps[1]) and torch.equal(reps[0].contiguous(), out), (name, v, i)
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
            REACHED.add(name)


# ------------------------------------------------------------------------------------------------ stem
def stem_model(x, w, pad, Ho, Wo):
    H, W = x.shape[2:]
    pb, pr = (Ho - 1) * 2 + 3 - H - pad, (Wo - 1) * 2 + 3 - W - pad
    return F.conv2d(F.pad(x, (pad, pr, pad, pb)), w, stride=2).permute(0, 2, 3, 1)


def test_stem_launches():
    L = _lib.lib()
    for v, i, (_, a, kw, out) in _launches("stem_raw"):
        x, w, (Ho, Wo), pad = a
        M, _, H, W = x.shape
        cout = w.shape[0]
        reps = []
        for _ in range(2):
            y = torch.full((M, Ho, Wo, cout), float("nan"), device=DEV)
            assert L.stp3_effnet_stem_raw(ptr(x), M, H, W, Ho, Wo, pad, pad, ptr(w.contiguous()), cout, ptr(y),
                                          stream()) == 0
            reps.append(y)
        torch.cuda.synchronize()
        assert torch.equal(reps[0], reps[1]) and torch.equal(reps[0], out)
        x64, w64 = x.double().cpu(), w.double().cpu()
        elementwise_ok(reps[0], stem_model(x64, w64, pad, Ho, Wo), stem_model(x64.abs(), w64.abs(), pad, Ho, Wo), 60)
        REACHED.add("stem_raw")
    for v, i, (_, a, kw, out) in _launches("stem_wgrad"):
        x, g, pad = a
        M, _, H, W = x.shape
        _, Ho, Wo, cout = g.shape
        nbytes = L.stp3_effnet_stem_wgrad_scratch_bytes(M, Ho, Wo, cout)
        reps = []
        for _ in range(2):
            dw = torch.full((cout, 3, 3, 3), float("nan"), device=DEV)
            scratch = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
            assert L.stp3_effnet_stem_wgrad(ptr(x), M, H, W, Ho, Wo, pad, pad, ptr(g), cout, ptr(dw), ptr(scratch),
                                            nbytes, stream()) == 0
            reps.append(dw)
        torch.cuda.synchronize()
        assert torch.equal(reps[0], reps[1]) and torch.equal(reps[0], out)
        wr = torch.zeros(cout, 3, 3, 3, dtype=torch.float64, requires_grad=True)
        exact, = torch.autograd.grad(stem_model(x.double().cpu(), wr, pad, Ho, Wo), [wr], g.double().cpu())
        wr = torch.zeros(cout, 3, 3, 3, dtype=torch.float64, requires_grad=True)
        mag, = torch.autograd.grad(stem_model(x.double().cpu().abs(), wr, pad, Ho, Wo), [wr], g.double().cpu().abs())
        reduction_ok(reps[0], exact, mag)
        REACHED.add("stem_wgrad")


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


def test_bn_act_launches():
    L = _lib.lib()
    for v, i, (_, a, kw, out) in _launches("bn_act"):
        x, st, gb = a[:3]
        swish = a[3] if len(a) > 3 else kw["swish"]
        mul, scale, res, hl = kw.get("mul"), kw.get("scale"), kw.get("res"), kw.get("hl", False)
        REACHED.add("bn_act" + (" swish" if swish else "") + (" stats" if st is not None else "") +
                    (" mul" if mul is not None else "") + (" scale" if scale is not None else "") +
                    (" res" if res is not None else "") + (" planes" if hl else ""))
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
        assert torch.equal(y0, y1) and torch.equal(y0, out[0])
        assert torch.equal(h0, h1) and torch.equal(h0, h2) and torch.equal(l0, l2)
        assert (h0[..., C:] == 0).all() and (l0[..., C:] == 0).all()
        if hl:
            assert torch.equal(h0, out[1].hi.view_as(h0)) and torch.equal(l0, out[1].lo.view_as(l0))
        REACHED.add("bn_act planes only")
        z, mag = _z64(x, st, gb)
        if swish:                                  # |swish'| <= 1.1
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


def test_bn_act_grad_launches():
    L = _lib.lib()
    for v, i, (_, a, kw, out) in _launches("bn_act_grad"):
        g, x, st, gb = a[:4]
        swish = a[4] if len(a) > 4 else kw["swish"]
        mul, add, scale = kw.get("mul"), kw.get("add"), kw.get("scale")
        REACHED.add("bn_act_grad" + (" swish" if swish else "") + (" mul" if mul is not None else "") +
                    (" add" if add is not None else "") + (" scale" if scale is not None else ""))
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
        assert torch.equal(reps[0], reps[1]) and torch.equal(reps[0], out)
        r, mag = g.double().cpu(), g.double().cpu().abs()
        if mul is not None:
            mv = mul.double().cpu().view(N, 1, 1, C)
            r, mag = r * mv, mag * mv.abs()
        if add is not None:
            av = add.double().cpu().view(N, 1, 1, C)
            r, mag = r + av, mag + av.abs()
        if swish:
            z, _ = _z64(x, st, gb)
            sg = torch.sigmoid(z)
            d = sg * (1 + z * (1 - sg))
            r, mag = r * d, mag * (sg * (1 + z.abs() * (1 - sg)))
        if scale is not None:
            sv = scale.double().cpu().view(N, 1, 1, 1)
            r, mag = r * sv, mag * sv.abs()
        # the recomputed z carries a few ulps of x's normalisation into swish'
        elementwise_ok(reps[0], r, mag, 64)


# ------------------------------------------------------------------------------------------------ squeeze-excite
def test_image_channel_dot_launches():
    L = _lib.lib()
    for v, i, (_, a, kw, out) in _launches("image_channel_dot"):
        y, u = a
        N, H, W, C = y.shape
        nbytes = L.stp3_image_channel_dot_scratch_bytes(N, H * W, C)
        reps = []
        for _ in range(2):
            o = torch.full((N, C), float("nan"), device=DEV)
            scratch = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
            assert L.stp3_image_channel_dot(ptr(y), ptr(u), N, H * W, C, ptr(o), ptr(scratch), nbytes, stream()) == 0
            reps.append(o)
        torch.cuda.synchronize()
        assert torch.equal(reps[0], reps[1]) and torch.equal(reps[0], out)
        p = y.double().cpu() * u.double().cpu()
        reduction_ok(reps[0], p.sum(dim=(1, 2)), p.abs().sum(dim=(1, 2)))
        REACHED.add("image_channel_dot")


def test_se_backward_launches():
    L = _lib.lib()
    for v, i, (_, a, kw, out) in _launches("se_backward"):
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
        assert all(torch.equal(p, q) and torch.equal(p, r) for p, q, r in zip(reps[0], reps[1], out))
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
            assert float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)) < 1e-5
        REACHED.add("se_backward")


# ------------------------------------------------------------------------------------------------ coverage
def test_every_entry_point_and_path_was_reached():
    for v in ("b0", "b4"):
        assert {r[0] for r in records(v)} == set(NAMES), v
    want = {"stem_raw", "stem_wgrad", "dw_raw", "dw_dgrad", "dw_wgrad", "image_channel_dot", "se_backward",
            "dw k3 s1", "dw k3 s2", "dw k5 s1", "dw k5 s2",
            "bn_act swish stats",                        # _bn0 / _bn1 / stem
            "bn_act swish stats planes",                 # the stem when block 0 expands, else absent
            "bn_act mul planes",                         # the gate
            "bn_act stats scale res planes",             # _bn2 with drop-connect and skip, feeding an expand
            "bn_act stats planes",                       # _bn2 without skip
            "bn_act stats scale res",                    # the last block's _bn2
            "bn_act planes only",
            "bn_act_grad swish", "bn_act_grad swish mul add", "bn_act_grad scale"}
    want.discard("bn_act swish stats planes")            # neither b0 nor b4 expands in block 0
    missing = want - REACHED
    assert not missing, missing
