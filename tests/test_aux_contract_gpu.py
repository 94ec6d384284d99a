"""GPU: every launch of the EfficientNet trunk kernels (stp3_effnet_stem, stp3_dw_fwd, stp3_se_gate) and of the dense
path's memory-bound helpers (stp3_f32_to_hilo, stp3_hilo_to_f32, stp3_spatial_sum, stp3_pool_bias, stp3_small_linear,
stp3_upsample2x_add) against the float64 reference of their contract (tests/aux_reference.py).

The launches are recorded from the model -- the dense wrappers and dense_train.to_hl replaced while it runs, each call's
inputs cloned and what production wrote cloned too: the b4 trunk on 18 images and the b0 trunk at 224 x 480, the
perceive forward with the fused and the unfused TemporalBlock tail, the stress shape, the encoder heads in eval, the
Prediction model (tests/test_conv_contract_gpu.py predict_model at 40 x 56, and _predict_hl at 200 x 200), and
train steps of the decoder, the DeepLab head, the TemporalModel, the encoder heads and the trainable trunk (b0 and b4 on
3 x 35 x 51 images, b4 on 6 x 224 x 480: stp3_se_gate asked for the gate with a one-row zero projection, to_hl at the
trunk's channel counts) -- and built synthetically for what
the model never passes (stem widths and pads, channel windows inside wider strides, one-pixel maps, squeeze-excite
projections whose last chunk is exactly 64 or 128 wide, rounding edge cases of the hi/lo split, multi-slice pooling
rows, 8-mod-16 upsample windows).  stp3_f32_to_plane (the one 16-bit plane of an autocast train step) is recorded from
the same train steps with their forward under torch.autocast in float16 and in bfloat16 (dense_train.to_hl with a
mode), and run synthetically in both layouts at the rounding edges of both types; every plane must be bitwise torch's
own .to(mode) of the input (NaN where torch has NaN), its padding +0.

Each launch is replayed twice through _lib.lib() into outputs filled with a sentinel (NaN for fp32, the bf16 NaN 0x7FA5
for planes) followed by a guard; scratch is 0xFF bytes (NaN), and the input channels a kernel must not read are NaN.
Checked per replay:
  - values against the fp64 reference, in units of fp32 ulps of the magnitudes of each value's terms (beyond the
    2^-17 split allowance where the output is a pair of bf16 planes), with the bars of BARS;
  - every stored plane pair a valid hi/lo split (hi a bf16 nearest to hi + lo): a wrongly rounded hi hides below the
    value bar;
  - padding channels exactly +0 where the header says they are written; every element outside the written window
    unchanged, including the guard; the stem, f32_to_hilo, the gate, the packed weights, sums and spatial sums fully
    written (no sentinel survives);
  - the two replays bitwise equal, and bitwise equal to what production wrote.  stp3_spatial_sum is the exception:
    it adds per-block partials with float atomics, so its sums are nondeterministic in the last bits and only the value
    bar applies to it.
The last test asserts that the replays reached every entry point and every listed feature, and prints the worst error of
each entry point."""
import ctypes
import itertools
import time
from dataclasses import dataclass, field
from typing import Optional

import pytest
import torch

from oracle import torch_dense as TD
from stp3_b200 import _lib, dense, dense_train
from tests import aux_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN = float("nan")
SENT16 = 0x7FA5            # bf16 NaN: the sentinel of every output plane element
GUARD = 64                 # sentinel elements after every output buffer
SPLIT = 2.0 ** -17         # what the hi/lo split of a stored value may lose
ULP = 2.0 ** -24

# Bars in fp32 ulps of the magnitudes of each value's terms (tests/aux_reference.py `mag`), about 4x the worst
# measured over every launch of this file on an H100 80GB HBM3 (700 W power limit; table in DESIGN.md section 4).  The
# squeeze-excite weights are held to their exact bound instead: 2^-17 (the split) + 2^-23 (the fp32 product) of
# |W_proj gate| with the kernel's own gate, i.e. a ratio of 1.
# stp3_spatial_sum sums each 128-pixel chunk in fp64, rounds it once and adds the chunks into each sum with float
# atomics, in no fixed order, so its round-off grows like the square root of the chunk count: its bar is
# BARS["spatial_sum"] up to SSUM_CHUNKS chunks per image (1.5 ulps at most measured there), and grows with
# sqrt(chunks / SSUM_CHUNKS) beyond (the Prediction model: 3.7 ulps at 18 chunks, bar 10.6; 9.9 at 313 chunks, bar 44).
BARS = {"stem": 16, "dw": 10, "dw sums": 10, "se gate": 4, "se weights": 1.0, "spatial_sum": 5,
        "pool_bias": 4, "small_linear": 16, "upsample": 6}
SSUM_CHUNKS = 4


def ssum_bar_scale(HW):
    return max(1.0, (-(-HW // 128) / SSUM_CHUNKS) ** 0.5)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    t = t.contiguous().reshape(-1)
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _planes_out(n):
    return [torch.full((n + GUARD,), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16) for _ in range(2)]


def _f32_out(n):
    return torch.full((n + GUARD,), NAN, dtype=torch.float32, device=DEV)


def _is_sent(t):
    return t.contiguous().view(torch.int16) == SENT16


def _poison(hi, lo, keep):
    """copies of planes (..., cs) whose channels outside the slice `keep` are the bf16 NaN sentinel"""
    out = []
    for p in (hi, lo):
        q = torch.full_like(p, 0).view(torch.int16).fill_(SENT16).view(torch.bfloat16)
        q[..., keep] = p[..., keep]
        out.append(q)
    return out


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    kind: str
    a: dict
    tag: str = ""
    prod: Optional[dict] = None            # what the production launch wrote, per window name
    features: set = field(default_factory=set)


def stem_case(x, w, b, Ho, Wo, pt, pl, ocs, tag, extra=()):
    n, _, H, W = x.shape
    cout = b.numel()
    f = {"stem", f"stem pad ({pt},{pl})", f"stem cout {cout}"} | set(extra)
    if n * Ho * Wo * (ocs // 16) % 256:
        f.add("stem ragged grid")
    if Ho * Wo == 1:
        f.add("stem one-pixel output")
    if H % 2 or W % 2:
        f.add("stem odd H or W")
    if ocs > 64:
        f.add("stem out_cstride 128")
    return Case("stem", dict(x=x, w=w.reshape(cout, 27).contiguous(), b=b, n=n, H=H, W=W, Ho=Ho, Wo=Wo, pt=pt, pl=pl,
                             cout=cout, ocs=ocs), tag, features=f)


def dw_case(xh, xl, w, b, k, s, pt, pl, Ho, Wo, ocs, sums, tag):
    n, H, W, ics = xh.shape
    C = b.numel()
    xh, xl = _poison(xh, xl, slice(0, C))
    f = {"dw", f"dw k{k} s{s}", "dw sums" if sums else "dw no sums"}
    if ics > C:
        f.add("dw in_cstride > C")
    if ics != ocs:
        f.add("dw in_cstride != out_cstride")
    if ocs > C:
        f.add("dw out_cstride > C")
    if pt != pl:
        f.add("dw pad_t != pad_l")
    if Ho == 1 or Wo == 1:
        f.add("dw Ho or Wo 1")
    if Ho % 8 or Wo % 16:
        f.add("dw ragged tiles")
    return Case("dw", dict(xh=xh, xl=xl, w=w, b=b, n=n, H=H, W=W, Ho=Ho, Wo=Wo, k=k, s=s, pt=pt, pl=pl, C=C, ics=ics,
                           ocs=ocs, sums=bool(sums)), tag, features=f)


def se_case(sums, C, inv_hw, w_r, b_r, w_e, b_e, w_p, tag, extra=()):
    n, ss = sums.shape
    R_, cout = w_r.shape[0], w_p.shape[0]
    if ss > C:
        sums = sums.clone()
        sums[:, C:] = NAN
    last = cout - (cout - 1) // 128 * 128
    f = {"se", f"se last chunk {128 if last > 64 else 64}", f"se {-(-cout // 128)} chunks"} | set(extra)
    if ss > C:
        f.add("se sums_stride > C")
    if C % 64:
        f.add("se C % 64 != 0")
    for v, name in ((n, "images"), (C, "C"), (R_, "R")):
        f.add(f"se {name} {v}")
    return Case("se", dict(sums=sums, ss=ss, n=n, C=C, inv_hw=inv_hw, w_r=w_r, b_r=b_r, R=R_, w_e=w_e, b_e=b_e,
                           w_p=w_p, cout=cout), tag, features=f)


def to_hilo_case(x, cl, n, C, H, W, cp, tag, extra=()):
    f = {"f32_to_hilo", f"f32_to_hilo {'NHWC' if cl else 'NCHW'}"} | set(extra)
    if cp > C:
        f.add("f32_to_hilo cp > C")
    if (H * W) % 32 or C % 32:
        f.add("f32_to_hilo ragged tiles")
    return Case("to_hilo", dict(x=x.reshape(-1), cl=int(cl), n=n, C=C, H=H, W=W, cp=cp), tag, features=f)


def to_plane_case(x, cl, n, C, H, W, cp, mode, tag, extra=()):
    name = "f16" if mode == torch.float16 else "bf16"
    f = {"f32_to_plane", f"f32_to_plane {name}", f"f32_to_plane {'NHWC' if cl else 'NCHW'}"} | set(extra)
    if cp > C:
        f.add("f32_to_plane cp > C")
    if C > 32:
        f.add("f32_to_plane several channel tiles")
    return Case("to_plane", dict(x=x.reshape(-1), cl=int(cl), n=n, C=C, H=H, W=W, cp=cp, mode=mode), tag, features=f)


def to_f32_case(hi, lo, n, H, W, c_off, C, tag):
    cs = hi.shape[-1]
    hi, lo = _poison(hi.reshape(n, H, W, cs), lo.reshape(n, H, W, cs), slice(c_off, c_off + C))
    f = {"hilo_to_f32"} | ({"hilo_to_f32 window"} if c_off or C < cs else set())
    return Case("to_f32", dict(hi=hi, lo=lo, n=n, H=H, W=W, cs=cs, c_off=c_off, C=C), tag, features=f)


def ssum_case(hi, lo, n, HW, tag, extra=()):
    cs = hi.shape[-1]
    return Case("ssum", dict(hi=hi.reshape(n, HW, cs), lo=lo.reshape(n, HW, cs), n=n, HW=HW, cs=cs), tag,
                features={"spatial_sum"} | ({"spatial_sum ragged chunk"} if HW % 128 else set()) | set(extra))


def pool_case(sums, T, C, inv_hw, temporal, cv, W1, b1, W2, bias, prior, acc, tag):
    n, ss = sums.shape
    nc = 0 if cv is None else cv.shape[1]
    R_, CO = W1.shape[0], W2.shape[0]
    if ss > C - nc:
        sums = sums.clone()
        sums[:, C - nc:] = NAN
    f = {"pool_bias", "pool_bias accumulate" if acc else "pool_bias bias" if bias is not None else "pool_bias bias NULL"}
    if temporal:
        f.add("pool_bias temporal" if T > 1 else "pool_bias temporal T 1")
    if nc:
        f.add("pool_bias n_const" + (" = C - 1" if nc == C - 1 else ""))
    if CO >= 64:
        f.add("pool_bias 4 row slices")
    if R_ == 1:
        f.add("pool_bias R 1")
    if C == 1:
        f.add("pool_bias C 1")
    if CO % 4:
        f.add("pool_bias CO % 4 != 0")
    return Case("pool", dict(sums=sums, ss=ss, n=n, T=T, C=C, inv_hw=inv_hw, temporal=bool(temporal), cv=cv, nc=nc,
                             W1=W1, b1=b1, R=R_, W2=W2, CO=CO, bias=bias, prior=prior, cos=prior.shape[1],
                             acc=bool(acc)), tag, features=f)


def lin_case(x, W, bias, prior, acc, tag):
    n, ci = x.shape
    co = W.shape[0]
    f = {"small_linear", "small_linear accumulate" if acc else "small_linear bias" if bias is not None
         else "small_linear bias NULL"}
    if co > 128:
        f.add("small_linear co > 128")
    if ci >= 1024:
        f.add("small_linear ci 1024")
    return Case("lin", dict(x=x, W=W, n=n, ci=ci, co=co, bias=bias, prior=prior, cos=prior.shape[1], acc=bool(acc)),
                tag, features=f)


def up_case(xh, xl, C, sh, sl, soff, ycs, yoff, tag):
    n, h, w, xcs = xh.shape
    xh, xl = _poison(xh, xl, slice(0, C))
    f = {"upsample2x_add", "upsample skip" if sh is not None else "upsample no skip"}
    scs = 0
    if sh is not None:
        scs = sh.shape[-1]
        sh, sl = _poison(sh, sl, slice(soff, soff + C))
        if soff % 16 == 8:
            f.add("upsample skip window 8 mod 16")
    if yoff % 16 == 8:
        f.add("upsample window 8 mod 16")
    if h == 1 or w == 1:
        f.add("upsample h or w 1")
    if C == 8:
        f.add("upsample C 8")
    return Case("up", dict(xh=xh, xl=xl, n=n, h=h, w=w, xcs=xcs, sh=sh, sl=sl, scs=scs, soff=soff, ycs=ycs, yoff=yoff,
                           C=C), tag, features=f)


# ------------------------------------------------------------------------------------------------ replay
def run(case: Case) -> dict:
    """one launch into fresh sentinel-filled outputs -> {name: whole output storage}"""
    L, a, k = _lib.lib(), case.a, case.kind
    ptr = lambda t: t.data_ptr() if t is not None else None          # noqa: E731
    if k == "stem":
        yh, yl = _planes_out(a["n"] * a["Ho"] * a["Wo"] * a["ocs"])
        code = L.stp3_effnet_stem(a["x"].data_ptr(), a["n"], a["H"], a["W"], a["Ho"], a["Wo"], a["pt"], a["pl"],
                                  a["w"].data_ptr(), a["b"].data_ptr(), a["cout"], a["ocs"], yh.data_ptr(),
                                  yl.data_ptr(), _stream())
        outs = {"hi": yh, "lo": yl}
    elif k == "dw":
        d = _lib.DwDesc(n_img=a["n"], H=a["H"], W=a["W"], Ho=a["Ho"], Wo=a["Wo"], k=a["k"], stride=a["s"],
                        pad_t=a["pt"], pad_l=a["pl"], C=a["C"], in_cstride=a["ics"], out_cstride=a["ocs"])
        nb = L.stp3_dw_sums_scratch_bytes(ctypes.byref(d))
        sc = torch.full((nb + 256,), 0xFF, dtype=torch.uint8, device=DEV)
        yh, yl = _planes_out(a["n"] * a["Ho"] * a["Wo"] * a["ocs"])
        sums = _f32_out(a["n"] * a["C"]) if a["sums"] else None
        code = L.stp3_dw_fwd(ctypes.byref(d), a["xh"].data_ptr(), a["xl"].data_ptr(), a["w"].data_ptr(),
                             a["b"].data_ptr(), yh.data_ptr(), yl.data_ptr(), ptr(sums), sc.data_ptr(), nb, _stream())
        outs = {"hi": yh, "lo": yl, "scratch": sc}
        if sums is not None:
            outs["sums"] = sums
    elif k == "se":
        elems = L.stp3_se_proj_weight_elems(a["C"], a["cout"])
        gate = _f32_out(a["n"] * a["C"])
        wi = torch.full((a["n"] * elems + GUARD,), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        code = L.stp3_se_gate(a["sums"].data_ptr(), a["ss"], a["n"], a["C"], a["inv_hw"], a["w_r"].data_ptr(),
                              a["b_r"].data_ptr(), a["R"], a["w_e"].data_ptr(), a["b_e"].data_ptr(), a["w_p"].data_ptr(),
                              a["cout"], gate.data_ptr(), wi.data_ptr(), _stream())
        outs = {"gate": gate, "w_img": wi}
    elif k == "to_hilo":
        yh, yl = _planes_out(a["n"] * a["H"] * a["W"] * a["cp"])
        code = L.stp3_f32_to_hilo(a["x"].data_ptr(), a["cl"], a["n"], a["C"], a["H"], a["W"], a["cp"], yh.data_ptr(),
                                  yl.data_ptr(), _stream())
        outs = {"hi": yh, "lo": yl}
    elif k == "to_plane":
        o = torch.full((a["n"] * a["H"] * a["W"] * a["cp"] + GUARD,), SENT16, dtype=torch.int16, device=DEV).view(a["mode"])
        code = L.stp3_f32_to_plane(a["x"].data_ptr(), a["cl"], a["n"], a["C"], a["H"], a["W"], a["cp"],
                                   dense.PLANE_OPERAND[a["mode"]], o.data_ptr(), _stream())
        outs = {"plane": o}
    elif k == "to_f32":
        o = _f32_out(a["n"] * a["C"] * a["H"] * a["W"])
        code = L.stp3_hilo_to_f32(a["hi"].data_ptr(), a["lo"].data_ptr(), a["n"], a["H"], a["W"], a["cs"], a["c_off"],
                                  a["C"], o.data_ptr(), _stream())
        outs = {"out": o}
    elif k == "ssum":
        o = _f32_out(a["n"] * a["cs"])
        code = L.stp3_spatial_sum(a["hi"].data_ptr(), a["lo"].data_ptr(), a["n"], a["HW"], a["cs"], o.data_ptr(), _stream())
        outs = {"sums": o}
    elif k == "pool":
        o = torch.cat([a["prior"].reshape(-1), torch.full((GUARD,), NAN, device=DEV)])
        code = L.stp3_pool_bias(a["sums"].data_ptr(), a["ss"], a["n"], a["T"], a["C"], a["inv_hw"], int(a["temporal"]),
                                ptr(a["cv"]), a["nc"], a["W1"].data_ptr(), a["b1"].data_ptr(), a["R"],
                                a["W2"].data_ptr(), a["CO"], ptr(a["bias"]), o.data_ptr(), a["cos"], int(a["acc"]),
                                _stream())
        outs = {"out": o}
    elif k == "lin":
        o = torch.cat([a["prior"].reshape(-1), torch.full((GUARD,), NAN, device=DEV)])
        code = L.stp3_small_linear(a["x"].data_ptr(), a["W"].data_ptr(), a["n"], a["ci"], a["co"], ptr(a["bias"]),
                                   o.data_ptr(), a["cos"], int(a["acc"]), _stream())
        outs = {"out": o}
    elif k == "up":
        yh, yl = _planes_out(a["n"] * 4 * a["h"] * a["w"] * a["ycs"])
        code = L.stp3_upsample2x_add(a["xh"].data_ptr(), a["xl"].data_ptr(), a["n"], a["h"], a["w"], a["xcs"],
                                     ptr(a["sh"]), ptr(a["sl"]), a["scs"], a["soff"], yh.data_ptr(), yl.data_ptr(),
                                     a["ycs"], a["yoff"], a["C"], _stream())
        outs = {"hi": yh, "lo": yl}
    else:
        raise AssertionError(k)
    _lib.check(code, f"replay {k}")
    torch.cuda.synchronize()
    return outs


def windows(case: Case, outs: dict) -> dict:
    """the elements the launch writes, per output, in the layout the recorder clones production's into"""
    a, k = case.a, case.kind
    if k == "to_plane":
        return {"plane": outs["plane"][:a["n"] * a["H"] * a["W"] * a["cp"]]}
    if k in ("stem", "to_hilo"):
        n = a["n"] * (a["Ho"] * a["Wo"] * a["ocs"] if k == "stem" else a["H"] * a["W"] * a["cp"])
        return {"hi": outs["hi"][:n], "lo": outs["lo"][:n]}
    if k == "dw":
        v = lambda t: t[:a["n"] * a["Ho"] * a["Wo"] * a["ocs"]].view(a["n"], a["Ho"], a["Wo"], a["ocs"])[..., :a["C"]]  # noqa: E731
        w = {"hi": v(outs["hi"]), "lo": v(outs["lo"])}
        if a["sums"]:
            w["sums"] = outs["sums"][:a["n"] * a["C"]]
        return w
    if k == "se":
        elems = _lib.lib().stp3_se_proj_weight_elems(a["C"], a["cout"])
        return {"gate": outs["gate"][:a["n"] * a["C"]], "w_img": outs["w_img"][:a["n"] * elems]}
    if k == "to_f32":
        return {"out": outs["out"][:a["n"] * a["C"] * a["H"] * a["W"]]}
    if k == "ssum":
        return {"sums": outs["sums"][:a["n"] * a["cs"]]}
    if k in ("pool", "lin"):
        co = a["CO"] if k == "pool" else a["co"]
        return {"out": outs["out"][:a["n"] * a["cos"]].view(a["n"], a["cos"])[:, :co]}
    if k == "up":
        v = lambda t: t[:a["n"] * 4 * a["h"] * a["w"] * a["ycs"]].view(a["n"], 2 * a["h"], 2 * a["w"], a["ycs"])[  # noqa: E731
            ..., a["yoff"]:a["yoff"] + a["C"]]
        return {"hi": v(outs["hi"]), "lo": v(outs["lo"])}
    raise AssertionError(k)


# ------------------------------------------------------------------------------------------------ checks
def _excess(hi, lo, ref, mag):
    """max over elements of the planes' error beyond the split allowance, in fp32 ulps of mag"""
    e = ((R.planes(hi, lo) - ref).abs() - SPLIT * ref.abs()).clamp_min(0)
    return float((e / (ULP * mag + 1e-300)).max()) if e.numel() else 0.0


def _ulps(got, ref, mag):
    return float(((got.double() - ref).abs() / (ULP * mag + 1e-300)).max()) if got.numel() else 0.0


def _guard_ok(t):
    g = t[-GUARD:]
    return bool(_is_sent(g).all()) if t.element_size() == 2 else bool(torch.isnan(g).all())


def _plane_checks(res, hi, lo, name=""):
    res[f"split{name}"] = bool(R.split_valid(hi, lo).all())


def check(case: Case) -> dict:
    """-> {"errs": {metric: error}, flag: bool, ...}; asserts nothing"""
    a, k = case.a, case.kind
    outs = run(case)
    outs2 = run(case)
    win = windows(case, outs)
    res = {"guard": all(_guard_ok(t) for nm, t in outs.items() if nm != "scratch")}
    if k != "ssum":     # float atomics: see the module docstring
        res["same"] = all(torch.equal(_bits(outs[nm]) if outs[nm].dtype != torch.uint8 else outs[nm],
                                      _bits(outs2[nm]) if outs2[nm].dtype != torch.uint8 else outs2[nm]) for nm in outs)
        if case.prod is not None:
            res["production"] = all(torch.equal(_bits(win[nm]), _bits(case.prod[nm])) for nm in case.prod)
    errs = {}
    if k == "stem":
        n, Ho, Wo, ocs, cout = a["n"], a["Ho"], a["Wo"], a["ocs"], a["cout"]
        hi, lo = (win[p].view(n, Ho, Wo, ocs) for p in ("hi", "lo"))
        ref = R.stem(a["x"], a["w"], a["b"], Ho, Wo, a["pt"], a["pl"], ocs)
        errs["stem"] = _excess(hi[..., :cout], lo[..., :cout], ref["y"][..., :cout], ref["mag"][..., :cout])
        res["written"] = not bool(_is_sent(hi).any() or _is_sent(lo).any())
        res["padding +0"] = not bool(_bits(hi[..., cout:]).any() or _bits(lo[..., cout:]).any())
        _plane_checks(res, hi, lo)
        res["saturated"] = float(ref["mag"].max()) > 90 if "stem swish saturates" in case.features else True
    elif k == "dw":
        n, Ho, Wo, ocs, C = a["n"], a["Ho"], a["Wo"], a["ocs"], a["C"]
        ref = R.dw(a["xh"], a["xl"], a["w"], a["b"], a["k"], a["s"], a["pt"], a["pl"], Ho, Wo, C)
        errs["dw"] = _excess(win["hi"], win["lo"], ref["y"], ref["mag"])
        _plane_checks(res, win["hi"], win["lo"])
        full = [outs[p][:n * Ho * Wo * ocs].view(n, Ho, Wo, ocs) for p in ("hi", "lo")]
        res["untouched"] = all(bool(_is_sent(t[..., C:]).all()) for t in full)
        res["written"] = not any(bool(_is_sent(win[p]).any()) for p in ("hi", "lo"))
        nb = outs["scratch"].numel() - 256
        if a["sums"]:
            res["sums written"] = not bool(torch.isnan(win["sums"]).any())
            errs["dw sums"] = _ulps(win["sums"].view(n, C), ref["sums"], ref["sums_mag"])
            res["scratch guard"] = bool((outs["scratch"][nb:] == 0xFF).all())
        else:
            res["scratch untouched"] = bool((outs["scratch"] == 0xFF).all())
    elif k == "se":
        n, C, cout = a["n"], a["C"], a["cout"]
        g = win["gate"].view(n, C)
        ref = R.se_gate(a["sums"], C, a["inv_hw"], a["w_r"], a["b_r"], a["w_e"], a["b_e"])
        res["gate written"] = not bool(torch.isnan(g).any())
        errs["se gate"] = float(((g.double() - ref["gate"]).abs() / (ULP * (ref["mag"] + 1))).max())
        elems = win["w_img"].numel() // n
        res["layout size"] = elems == R.se_layout(C, cout)[1]
        hi, lo = R.se_unpack(win["w_img"].view(n, elems), C, cout)
        wref = R.se_weights(a["w_p"], g, C, cout)
        val = R.planes(hi, lo)
        errs["se weights"] = float(((val - wref).abs() / ((SPLIT + 2.0 ** -23) * wref.abs() + 1e-300)).max())
        pad = torch.ones_like(wref, dtype=torch.bool)
        pad[:, :cout, :C] = False
        res["padding +0"] = not bool(_bits(hi[pad]).any() or _bits(lo[pad]).any())
        res["written"] = not bool(_is_sent(win["w_img"]).any())
        _plane_checks(res, hi, lo)
    elif k == "to_hilo":
        hi, lo = R.f32_to_hilo(a["x"], a["cl"], a["n"], a["C"], a["H"], a["W"], a["cp"])
        res["bitwise"] = torch.equal(_bits(win["hi"]), _bits(hi)) and torch.equal(_bits(win["lo"]), _bits(lo))
    elif k == "to_plane":
        ref = R.f32_to_plane(a["x"], a["cl"], a["n"], a["C"], a["H"], a["W"], a["cp"], a["mode"]).reshape(-1)
        got = win["plane"]
        nan = torch.isnan(ref)
        res["nan"] = torch.equal(torch.isnan(got), nan)
        res["bitwise"] = torch.equal(_bits(got)[~nan], _bits(ref)[~nan])
    elif k == "to_f32":
        ref = R.hilo_to_f32(a["hi"], a["lo"], a["n"], a["H"], a["W"], a["cs"], a["c_off"], a["C"])
        res["bitwise"] = torch.equal(_bits(win["out"]), _bits(ref))
    elif k == "ssum":
        ref = R.spatial_sum(a["hi"], a["lo"], a["n"], a["HW"], a["cs"])
        res["written"] = not bool(torch.isnan(win["sums"]).any())
        errs["spatial_sum"] = _ulps(win["sums"].view(a["n"], a["cs"]), ref["sums"], ref["mag"])
        res["bar scale"] = ssum_bar_scale(a["HW"])
    elif k in ("pool", "lin"):
        if k == "pool":
            ref = R.pool_bias(a["sums"], a["n"], a["T"], a["C"], a["inv_hw"], a["temporal"], a["cv"], a["nc"], a["W1"],
                              a["b1"], a["W2"], a["bias"], a["prior"], a["acc"])
            co = a["CO"]
        else:
            ref = R.small_linear(a["x"], a["W"], a["bias"], a["prior"], a["acc"])
            co = a["co"]
        errs["pool_bias" if k == "pool" else "small_linear"] = _ulps(win["out"], ref["out"], ref["mag"])
        rows = outs["out"][:a["n"] * a["cos"]].view(a["n"], a["cos"])
        res["untouched"] = torch.equal(_bits(rows[:, co:]), _bits(a["prior"][:, co:]))
    elif k == "up":
        ref = R.upsample2x_add(a["xh"], a["xl"], a["n"], a["h"], a["w"], a["C"], a["sh"], a["sl"], a["soff"])
        errs["upsample"] = _excess(win["hi"], win["lo"], ref["y"], ref["mag"])
        _plane_checks(res, win["hi"], win["lo"])
        full = [outs[p][:a["n"] * 4 * a["h"] * a["w"] * a["ycs"]].view(a["n"], 2 * a["h"], 2 * a["w"], a["ycs"])
                for p in ("hi", "lo")]
        res["untouched"] = all(bool(_is_sent(t[..., :a["yoff"]]).all() and _is_sent(t[..., a["yoff"] + a["C"]:]).all())
                               for t in full)
    res["errs"] = errs
    return res


def passed(res):
    return all(v for v in res.values() if isinstance(v, bool)) and all(e <= BARS[m] * res.get("bar scale", 1.0)
                                                                       for m, e in res["errs"].items())


# ------------------------------------------------------------------------------------------------ recording
def _hl_flat(h: dense.HL):
    B, T, H, W, cs = h.hi.shape
    return h.hi.reshape(B * T, H, W, cs).clone(), h.lo.reshape(B * T, H, W, cs).clone()


class Recorder:
    """Replaces the dense wrappers of the nine entry points (and dense_train.to_hl) while the model runs; every call
    becomes a Case with cloned inputs and a clone of what production wrote."""
    NAMES = ("effnet_stem", "dw_conv", "se_gate", "from_f32", "to_f32", "spatial_sum", "pool_bias", "small_linear",
             "upsample2x_add")

    def __init__(self, source):
        self.source, self.cases = source, []

    def __enter__(self):
        self.mp = pytest.MonkeyPatch()
        for nm in self.NAMES:
            self.mp.setattr(dense, nm, getattr(self, "_" + nm)(getattr(dense, nm)))
        self.mp.setattr(dense_train, "to_hl", self._to_hl(dense_train.to_hl))
        return self

    def __exit__(self, *exc):
        self.mp.undo()
        torch.cuda.synchronize()

    def _add(self, case, prod):
        case.tag = f"{self.source}: {case.tag}"
        case.prod = {k: v.detach().clone() for k, v in prod.items()} if prod is not None else None
        case.features |= {"recorded", f"recorded {case.kind}"}
        self.cases.append(case)

    def _effnet_stem(self, orig):
        def f(x, w, b, out_hw, pad, cp=dense.KB):
            xs = x.detach().float().contiguous().clone()
            out = orig(x, w, b, out_hw, pad, cp)
            self._add(stem_case(xs, w.clone(), b.clone(), *out_hw, *pad, cp, f"stem {tuple(xs.shape)}"),
                      {"hi": out.hi.reshape(-1), "lo": out.lo.reshape(-1)})
            return out
        return f

    def _dw_conv(self, orig):
        def f(x, w, b, k, stride, pad, out_hw, out=None, sums=None):
            xh, xl = _hl_flat(x)
            y = orig(x, w, b, k, stride, pad, out_hw, out=out, sums=sums)
            C = b.numel()
            prod = {"hi": y.hi[..., :C].reshape(-1), "lo": y.lo[..., :C].reshape(-1)}
            if sums is not None:
                prod["sums"] = sums.reshape(-1)
            self._add(dw_case(xh, xl, w.clone(), b.clone(), k, stride, *pad, *out_hw, y.hi.shape[-1], sums is not None,
                              f"dw k{k} s{stride} C{C} {tuple(xh.shape[:3])}"), prod)
            return y
        return f

    def _se_gate(self, orig):
        def f(sums, hw, C, w_r, b_r, w_e, b_e, w_proj, gate=None):
            sc = sums.clone()
            # the train-mode trunk asks for the gate and passes one zero projection row it does not use
            extra = ("se gate output, one-row projection",) if gate is not None and w_proj.shape[0] == 1 else ()
            if gate is None:
                gate = torch.empty((sums.shape[0], C), dtype=torch.float32, device=sums.device)
            w_img = orig(sums, hw, C, w_r, b_r, w_e, b_e, w_proj, gate=gate)
            self._add(se_case(sc, C, 1.0 / hw, w_r.clone(), b_r.clone(), w_e.clone(), b_e.clone(), w_proj.clone(),
                              f"se C{C} R{w_r.shape[0]} cout{w_proj.shape[0]} n{sums.shape[0]}", extra),
                      {"gate": gate.reshape(-1), "w_img": w_img.reshape(-1)})
            return w_img
        return f

    def _from_f32(self, orig):
        def f(x, channels_last=False, cp=None):
            xs = x.detach().float().contiguous().clone()
            out = orig(x, channels_last, cp)
            B, T, H, W, cpo = out.hi.shape
            C = xs.shape[-1] if channels_last else xs.shape[2]
            self._add(to_hilo_case(xs, channels_last, B * T, C, H, W, cpo, f"from_f32 {tuple(xs.shape)} cp{cpo}"),
                      {"hi": out.hi.reshape(-1), "lo": out.lo.reshape(-1)})
            return out
        return f

    def _to_hl(self, orig):
        def f(x, cp=None, mode=None):
            xs = x.clone()
            out = orig(x, cp, **dense_train.amp_kw(mode))
            N, H, W, C = xs.shape
            if mode is not None:
                self._add(to_plane_case(xs, 1, N, C, H, W, out.hi.shape[-1], mode, f"to_hl {tuple(xs.shape)} {mode}",
                                        ("to_hl plane",)), {"plane": out.hi.reshape(-1)})
                return out
            extra = ("to_hl",) + (("to_hl C % 64 != 0",) if C % 64 else ()) + (("to_hl C > 512",) if C > 512 else ())
            self._add(to_hilo_case(xs, 1, N, C, H, W, out.hi.shape[-1], f"to_hl {tuple(xs.shape)}", extra),
                      {"hi": out.hi.reshape(-1), "lo": out.lo.reshape(-1)})
            return out
        return f

    def _to_f32(self, orig):
        def f(x, c_off=0, c=None):
            hi, lo = _hl_flat(x)
            out = orig(x, c_off, c)
            n, H, W, _ = hi.shape
            C = c if c is not None else x.c
            self._add(to_f32_case(hi, lo, n, H, W, c_off, C, f"to_f32 {tuple(hi.shape)} [{c_off}, +{C})"),
                      {"out": out.reshape(-1)})
            return out
        return f

    def _spatial_sum(self, orig):
        def f(x):
            hi, lo = _hl_flat(x)
            out = orig(x)
            n, H, W, _ = hi.shape
            self._add(ssum_case(hi, lo, n, H * W, f"spatial_sum {tuple(hi.shape)}"), None)
            return out
        return f

    def _pool_bias(self, orig):
        def f(sums, T, C, hw, temporal, W1, b1, W2, out, accumulate, const=None, bias=None):
            args = [t.clone() if t is not None else None for t in (sums, W1, b1, W2, out, const, bias)]
            orig(sums, T, C, hw, temporal, W1, b1, W2, out, accumulate, const=const, bias=bias)
            s, w1, bb1, w2, prior, cv, bs = args
            self._add(pool_case(s, T, C, 1.0 / hw, temporal, cv, w1, bb1, w2, bs, prior, accumulate,
                                f"pool_bias C{C} R{W1.shape[0]} CO{W2.shape[0]} T{T} n{sums.shape[0]}"),
                      {"out": out[:, :W2.shape[0]]})
        return f

    def _small_linear(self, orig):
        def f(x, W, out, accumulate, bias=None):
            args = [t.clone() if t is not None else None for t in (x, W, out, bias)]
            orig(x, W, out, accumulate, bias=bias)
            xs, ws, prior, bs = args
            self._add(lin_case(xs, ws, bs, prior, accumulate, f"small_linear {tuple(xs.shape)} -> {W.shape[0]}"),
                      {"out": out[:, :W.shape[0]]})
        return f

    def _upsample2x_add(self, orig):
        def f(x, skip, c, skip_coff=0, out=None, out_coff=0):
            xh, xl = _hl_flat(x)
            sh, sl = _hl_flat(skip) if skip is not None else (None, None)
            y = orig(x, skip, c, skip_coff=skip_coff, out=out, out_coff=out_coff)
            w = slice(out_coff, out_coff + c)
            self._add(up_case(xh, xl, c, sh, sl, skip_coff, y.hi.shape[-1], out_coff,
                              f"upsample {tuple(xh.shape)} C{c} @{out_coff}/{y.hi.shape[-1]}"),
                      {"hi": y.hi[..., w].reshape(-1), "lo": y.lo[..., w].reshape(-1)})
            return y
        return f


# ------------------------------------------------------------------------------------------------ the models' launches
def rec_trunk(version, n_img):
    from oracle import efficientnet_oracle as EO
    from stp3_b200.models import efficientnet as EN
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=7), version)
    nat = EN.EfficientNetTrunk(version)
    nat.load_state_dict(ora.state_dict(), strict=True)
    nat = nat.to(DEV)
    x = torch.randn(n_img, 3, 224, 480, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad(), Recorder(f"trunk {version} {n_img}x224x480") as r:
        nat(x)
    return r.cases


def rec_perceive(block_fused):
    from stp3_b200.utils import synthetic as syn
    from tests import test_conv_contract_gpu as CC
    mp = pytest.MonkeyPatch()
    mp.setenv("STP3_BLOCK_FUSED", block_fused)
    try:
        with torch.no_grad():
            model, lcfg = CC._stp3_model(64, 3, [-10.0, 10.0, 0.5], [-14.0, 14.0, 0.5])
            inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
            with Recorder(f"perceive fused={block_fused}") as r:
                model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                       inp["extrinsics"], inp["future_egomotion"])
    finally:
        mp.undo()
    return r.cases


def rec_stress():
    from stp3_b200.utils import synthetic as syn
    from tests import test_conv_contract_gpu as CC
    with torch.no_grad():
        model, lcfg = CC._stp3_model(128, 5, [-8.0, 8.0, 0.5], [-8.0, 8.0, 0.5])
        inp = syn.lift_inputs(lcfg, 1, seed=5, random_pose=True)
        with Recorder("stress C128 S5") as r:
            model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                   inp["extrinsics"], inp["future_egomotion"])
    return r.cases


def rec_predict_small(carla):
    """the Prediction model's forward at 40 x 56, B = 2 (tests/test_conv_contract_gpu.py predict_model): the present
    distribution's spatial sums on 3 x 4 maps and its small_linear with 1 / (h w) folded into the weights"""
    from tests import test_conv_contract_gpu as CC
    r = Recorder(f"predict {'carla' if carla else 'nuscenes'} 40x56")
    CC.run_predict_small(carla, r)
    return r.cases


def rec_predict_200():
    """STP3._predict_hl on (1, 3, 64, 200, 200) present states: the distribution's sums on 13 x 13 maps"""
    from tests import test_conv_contract_gpu as CC
    r = Recorder("predict 200x200")
    CC.run_predict_200(r)
    return r.cases


def rec_encoder_heads():
    from oracle.make_golden_dense import dense_input
    from stp3_b200.config import get_cfg
    from stp3_b200.models.encoder import Encoder
    with torch.no_grad():
        enc = TD.init_exact(Encoder(get_cfg().MODEL.ENCODER, D=48, backbone=torch.nn.Identity()), seed=11).eval().to(DEV)
        r_hi, r_lo = dense_input((2, 160, 14, 30), 21).to(DEV), dense_input((2, 56, 28, 60), 22).to(DEV)
        with Recorder("encoder heads eval") as r:
            enc.heads_hl(r_lo, r_hi)
    return r.cases


def rec_amp(mode, step, *args):
    """a train step of tests/test_train_contract_gpu.py with its forward under torch.autocast(dtype=mode)"""
    from tests import test_train_contract_gpu as TC
    with Recorder(f"{step} {mode}") as r:
        getattr(TC, step)(*args, mode=mode)
    return r.cases


def rec_train_trunk(name):
    """a train step of the trainable trunk (tests/test_train_contract_gpu.py trunk_step): stp3_se_gate asked for the
    gate with a one-row zero projection, and to_hl of the projections' and expand convolutions' gradients"""
    from tests import test_train_contract_gpu as TC
    with Recorder(f"train {name}") as r:
        TC.trunk_step(*TC.TRUNK_STEPS[name])
    return r.cases


def rec_train(name, fn, *args):
    """a train step of the model of tests/test_train_contract_gpu.py (its own recorder runs too, unused)"""
    from tests import test_train_contract_gpu as TC
    with Recorder(f"train {name}") as r:
        getattr(TC, fn)(*args)
    return r.cases


# ------------------------------------------------------------------------------------------------ synthetic launches
def rnd(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def planes_of(x_cl, cs):
    """(n, H, W, C) fp32 -> hi/lo planes (n, H, W, cs), channels [C, cs) zero"""
    full = torch.zeros(*x_cl.shape[:-1], cs, device=DEV)
    full[..., :x_cl.shape[-1]] = x_cl
    hi, lo = R.split(full)
    return hi.contiguous(), lo.contiguous()


def synth_stem():
    cases = []

    def add(n, H, W, cout, pt, pl, ocs, tag, scale=1.0, extra=()):
        s = len(cases)
        x = rnd(n, 3, H, W, seed=100 + s, scale=scale)
        w, b = rnd(cout, 27, seed=200 + s, scale=0.3), rnd(cout, seed=300 + s, scale=0.1)
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        cases.append(stem_case(x, w, b, Ho, Wo, pt, pl, ocs, tag, extra))
    for i, cout in enumerate((1, 8, 24, 32, 40, 63, 64)):
        add(2, 15 + 2 * i, 22 + i, cout, i % 3, (i + 1) % 3, 128, f"cout {cout}, out_cstride 128")
    for pt, pl in itertools.product(range(3), range(3)):
        add(1, 17, 23, 32, pt, pl, 64, f"pads ({pt}, {pl}), odd H and W")
    add(3, 1, 1, 40, 1, 1, 64, "one-pixel outputs")
    add(1, 13, 17, 48, 0, 1, 64, "252 threads: ragged last block")
    add(2, 16, 20, 24, 1, 0, 64, "|a| > 90: swish saturates", scale=300.0, extra=("stem swish saturates",))
    return cases


def synth_dw():
    cases = []
    specs = [  # k, s, pt, pl, C, ics, ocs, H, W, sums
        (3, 1, 0, 2, 8, 64, 128, 13, 21, True), (3, 2, 2, 0, 56, 128, 64, 17, 33, False),
        (5, 1, 4, 1, 72, 128, 192, 9, 19, True), (5, 2, 1, 4, 200, 256, 256, 23, 37, True),
        (3, 1, 1, 1, 8, 64, 64, 1, 29, True), (5, 2, 3, 2, 56, 64, 128, 31, 1, True),
        (3, 2, 1, 0, 72, 192, 128, 2, 2, False), (5, 1, 0, 3, 200, 256, 256, 12, 50, False),
        (3, 1, 2, 1, 64, 64, 64, 40, 70, True), (5, 2, 2, 2, 8, 128, 64, 1, 1, True)]
    for i, (k, s, pt, pl, C, ics, ocs, H, W, sums) in enumerate(specs):
        n = 2 if i % 2 else 3
        xh, xl = planes_of(rnd(n, H, W, C, seed=400 + i), ics)
        w, b = rnd(k * k, C, seed=500 + i, scale=1.0 / k), rnd(C, seed=600 + i, scale=0.1)
        Ho, Wo = max((H + 2 * pt - k) // s + 1, 1), max((W + 2 * pl - k) // s + 1, 1)
        cases.append(dw_case(xh, xl, w, b, k, s, pt, pl, Ho, Wo, ocs, sums,
                             f"k{k} s{s} pad ({pt},{pl}) C{C} in {ics} out {ocs} {H}x{W} -> {Ho}x{Wo}"))
    return cases


def synth_se():
    cases = []
    for i, (C, R_, cout, n, extra) in enumerate([(8, 1, 1, 1, 0), (65, 4, 63, 73, 7), (65, 1024, 64, 3, 0),
                                                 (8, 2, 65, 73, 8), (4096, 16, 128, 2, 64), (65, 8, 129, 5, 3),
                                                 (4096, 1024, 192, 1, 0), (8, 1, 193, 73, 0), (65, 3, 256, 1, 63),
                                                 (65, 5, 300, 2, 0)]):
        hw = 49
        sums = rnd(n, C + extra, seed=700 + i, scale=0.5 * hw)
        cases.append(se_case(sums, C, 1.0 / hw, rnd(R_, C, seed=710 + i, scale=C ** -0.5), rnd(R_, seed=720 + i, scale=0.1),
                             rnd(C, R_, seed=730 + i, scale=R_ ** -0.5), rnd(C, seed=740 + i, scale=0.1),
                             rnd(cout, C, seed=750 + i, scale=C ** -0.5),
                             f"C{C} R{R_} cout{cout} n{n} sums_stride {C + extra}"))
    return cases


def _specials(n):
    """fp32 values at the edges of the split: +-0, fp32 and bf16 subnormals, the largest bf16, values that round to it
    or overflow past it, exact ties of the hi rounding"""
    v = torch.tensor([0.0, -0.0, 1e-45, -3e-42, 1e-39, -1.1754942e-38, 9.2e-41, 3.3895314e38, -3.3895314e38,
                      3.3910e38, 3.3961e38, -3.4028235e38, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8 + 2 ** -20),
                      65504.0, 1e-30, -2.5e-20], dtype=torch.float32)
    return v.repeat(-(-n // v.numel()))[:n]


def synth_hilo():
    cases = []
    for i, (n, C, H, W, cp, cl, special) in enumerate([(2, 37, 5, 7, 64, 0, False), (2, 37, 5, 7, 64, 1, False),
                                                       (3, 64, 4, 8, 64, 0, False), (1, 100, 9, 13, 192, 1, True),
                                                       (2, 13, 3, 11, 64, 0, True), (1, 8, 1, 1, 64, 1, False)]):
        x = rnd(n * C * H * W, seed=800 + i, scale=3.0)
        if special:
            x[::3] = _specials(x[::3].numel()).to(DEV)
        cases.append(to_hilo_case(x, cl, n, C, H, W, cp, f"{'NHWC' if cl else 'NCHW'} n{n} C{C} {H}x{W} cp{cp}",
                                  ("f32_to_hilo edge values",) if special else ()))
    for i, (n, H, W, cs, c_off, C) in enumerate([(2, 5, 7, 64, 8, 37), (1, 1, 1, 128, 64, 64), (1, 9, 13, 192, 0, 100),
                                                 (3, 3, 11, 64, 0, 64)]):
        hi, lo = planes_of(rnd(n, H, W, cs, seed=900 + i), cs)
        cases.append(to_f32_case(hi, lo, n, H, W, c_off, C, f"n{n} {H}x{W} [{c_off}, +{C}) of {cs}"))
    for i, (n, HW, cs) in enumerate([(3, 35, 8), (1, 1, 64), (2, 300, 1024), (4, 129, 200)]):
        hi, lo = planes_of(rnd(n, HW, 1, cs, seed=1000 + i, scale=4.0), cs)
        cases.append(ssum_case(hi, lo, n, HW, f"n{n} HW{HW} cs{cs}"))
    # 1 at the first pixel, then 299 terms of 0.75 ulp(1) / 2: an fp32 running sum drops every one of them (95 ulps of
    # the total in the first chunk), a chunk summed exactly loses at most one rounding
    x = torch.full((2, 300, 1, 64), 1.5 * 2.0 ** -25, device=DEV)
    x[:, 0] = 1.0
    x[1] *= -1.0
    hi, lo = planes_of(x, 64)
    cases.append(ssum_case(hi, lo, 2, 300, "n2 HW300 cs64: small terms after a large one",
                           ("spatial_sum small terms after a large one",)))
    return cases


def _plane_specials(mode):
    """fp32 values at the rounding edges of `mode`: ties to even, subnormals and values below half the smallest one,
    the largest finite value and the first values that round past it, -0.0, NaN and +-inf"""
    inf, nan = float("inf"), float("nan")
    both = [0.0, -0.0, nan, inf, -inf, 1.0, -1.0, 3.0e-39, -1e-45]
    if mode == torch.float16:
        v = [1 + 2 ** -11, 1 + 3 * 2 ** -11, -(1 + 2 ** -11), 2 ** -24, 3 * 2 ** -25, 2 ** -25, 2 ** -25 * (1 + 2 ** -20),
             -2 ** -26, 2 ** -26, 5 * 2 ** -26, 2 ** -14 - 2 ** -25, 65504.0, 65519.0, 65520.0, -65520.0, 1e6, 2.0 ** -15]
    else:
        v = [1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 1e-45, -3e-42, 1e-39, 9.2e-41, 1.1754942e-38,
             3.3895314e38, -3.3895314e38, 3.3961e38, 3.3962e38, -3.4e38, 3.4028235e38, 1.0 + 2 ** -8 + 2 ** -20]
    return torch.tensor(both + v, dtype=torch.float32)


def synth_plane():
    cases = []
    for mode in (torch.float16, torch.bfloat16):
        sp = _plane_specials(mode)
        for i, (n, C, H, W, cp, cl) in enumerate([(2, 37, 5, 7, 64, 0), (2, 37, 5, 7, 64, 1), (3, 64, 4, 8, 64, 0),
                                                  (1, 100, 9, 13, 192, 1), (1, 100, 9, 13, 128, 0), (1, 8, 1, 1, 64, 1)]):
            x = rnd(n * C * H * W, seed=1400 + i, scale=30.0)
            x[::2] = sp.repeat(-(-x[::2].numel() // sp.numel()))[:x[::2].numel()].to(DEV)
            cases.append(to_plane_case(x, cl, n, C, H, W, cp, mode, f"{'NHWC' if cl else 'NCHW'} n{n} C{C} {H}x{W} "
                                       f"cp{cp} {mode}", ("f32_to_plane edge values",)))
    return cases


def synth_small():
    cases = []
    for i, (B, T, C, R_, CO, nc, temporal, with_bias, acc, extra) in enumerate([
            (2, 3, 70, 35, 130, 0, True, True, False, 8), (6, 1, 64, 16, 64, 0, True, False, False, 0),
            (2, 3, 1, 1, 1, 0, True, True, True, 0), (2, 2, 9, 7, 63, 8, False, True, False, 3),
            (1, 4, 40, 12, 65, 2, True, False, True, 5), (3, 2, 20, 1, 5, 0, False, False, False, 0)]):
        n, hw = B * T, 37 * 29
        sums = rnd(n, C - nc + extra, seed=1100 + i, scale=float(hw))
        cv = rnd(n, nc, seed=1110 + i) if nc else None
        W1, b1, W2 = rnd(R_, C, seed=1120 + i, scale=0.2), rnd(R_, seed=1130 + i), rnd(CO, R_, seed=1140 + i, scale=0.2)
        bias = rnd(CO + 3, seed=1150 + i) if with_bias else None
        prior = rnd(n, CO + 3, seed=1160 + i) if acc else torch.full((n, CO + 3), NAN, device=DEV)
        cases.append(pool_case(sums, T, C, 1.0 / hw, temporal, cv, W1, b1, W2, bias, prior, acc,
                               f"B{B} T{T} C{C} R{R_} CO{CO} n_const {nc} temporal {temporal} acc {acc}"))
    for i, (n, ci, co, with_bias, acc) in enumerate([(3, 1024, 300, True, False), (2, 6, 129, False, True),
                                                     (5, 17, 1, False, False), (1, 1, 64, True, False)]):
        prior = rnd(n, co + 5, seed=1260 + i) if acc else torch.full((n, co + 5), NAN, device=DEV)
        cases.append(lin_case(rnd(n, ci, seed=1200 + i), rnd(co, ci, seed=1210 + i, scale=ci ** -0.5),
                              rnd(co, seed=1220 + i) if with_bias else None, prior, acc,
                              f"n{n} ci{ci} co{co} bias {with_bias} acc {acc}"))
    for i, (n, h, w, C, xcs, skip, scs, soff, ycs, yoff) in enumerate([
            (2, 1, 5, 8, 64, True, 64, 8, 64, 24), (1, 4, 1, 16, 64, False, 0, 0, 128, 40),
            (3, 3, 6, 40, 64, True, 128, 72, 192, 136), (1, 1, 1, 64, 64, False, 0, 0, 64, 0),
            (2, 5, 7, 8, 128, True, 64, 56, 64, 8)]):
        xh, xl = planes_of(rnd(n, h, w, C, seed=1300 + i), xcs)
        sh, sl = planes_of(rnd(n, 2 * h, 2 * w, scs, seed=1310 + i), scs) if skip else (None, None)
        cases.append(up_case(xh, xl, C, sh, sl, soff, ycs, yoff,
                             f"n{n} {h}x{w} C{C} skip {skip} @{soff}/{scs} -> @{yoff}/{ycs}"))
    return cases


GATES_ALL = dict(perceive_hdmap=True, predict_pedestrian=True, predict_instance=True, predict_future_flow=True,
                 planning=True)

SOURCES = {
    "trunk_b4": lambda: rec_trunk("b4", 18),
    "trunk_b0": lambda: rec_trunk("b0", 6),
    "perceive_fused": lambda: rec_perceive("1"),
    "perceive_unfused": lambda: rec_perceive("0"),
    "stress": rec_stress,
    "encoder_heads_eval": rec_encoder_heads,
    "predict_small_nuscenes": lambda: rec_predict_small(False),
    "predict_small_carla": lambda: rec_predict_small(True),
    "predict_200x200": rec_predict_200,
    "train_decoder": lambda: rec_train("decoder 48x64", "rec_decoder", (2, 3, 64, 48, 64), GATES_ALL, "d"),
    "train_deeplab": lambda: rec_train("deeplab 48x64", "rec_deeplab", 64, 64, 128, 6, 48, 64, "h"),
    "train_temporal": lambda: rec_train("temporal 48x64", "rec_temporal", 70, 6, 3, 2, 48, 64, "t"),
    "train_encoder_heads_feat": lambda: rec_train("encoder heads feat", "rec_encoder_heads", "feat"),
    "train_encoder_heads_uc": lambda: rec_train("encoder heads uc", "rec_encoder_heads", "uc"),
    "synthetic_stem": synth_stem,
    "synthetic_dw": synth_dw,
    "synthetic_se": synth_se,
    "synthetic_hilo": synth_hilo,
    "synthetic_small": synth_small,
    "synthetic_plane": synth_plane,
    "train_trunk_b0_35x51": lambda: rec_train_trunk("trunk_b0_35x51"),
    "train_trunk_b4_35x51": lambda: rec_train_trunk("trunk_b4_35x51"),
    "train_trunk_b4_224x480": lambda: rec_train_trunk("trunk_b4_224x480"),
}
for _m, _nm in ((torch.float16, "fp16"), (torch.bfloat16, "bf16")):
    SOURCES.update({
        f"amp_decoder_{_nm}": lambda m=_m: rec_amp(m, "decoder_step", (2, 3, 64, 48, 64), GATES_ALL),
        f"amp_deeplab_{_nm}": lambda m=_m: rec_amp(m, "deeplab_step", 64, 64, 128, 6, 48, 64),
        f"amp_temporal_{_nm}": lambda m=_m: rec_amp(m, "temporal_step", 70, 6, 3, 2, 48, 64),
        f"amp_encoder_heads_{_nm}": lambda m=_m: rec_amp(m, "encoder_heads_step", "feat")})

_RUNS = {}


def run_source(name):
    if name in _RUNS:
        return _RUNS[name]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    cases = SOURCES[name]()
    assert cases, f"{name}: no launch recorded"
    rows = []
    for c in cases:
        r = check(c)
        rows.append(dict(kind=c.kind, tag=c.tag, features=set(c.features), res=r, ok=passed(r)))
    del cases
    torch.cuda.empty_cache()
    print(f"\n{name}: {len(rows)} launches in {time.time() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated")
    _RUNS[name] = rows
    return rows


def _fmt(r):
    res = r["res"]
    s = " ".join(f"{m} {e:.3g}" for m, e in res["errs"].items())
    flags = [k for k, v in res.items() if isinstance(v, bool) and not v]
    return f"  {r['kind']:<8s} {r['tag'][:80]:<80s} {s}" + (f"  FAILED {flags}" if flags else "")


@pytest.mark.parametrize("name", list(SOURCES))
def test_aux_launches_against_the_fp64_contract(name):
    rows = run_source(name)
    for r in rows:
        print(_fmt(r))
    bad = [_fmt(r) for r in rows if not r["ok"]]
    assert not bad, "\n".join(bad)


REQUIRED = (["recorded"] + [f"recorded {k}" for k in ("stem", "dw", "se", "to_hilo", "to_f32", "ssum", "pool", "lin", "up")]
            + ["to_hl", "to_hl plane", "recorded to_plane", "to_hl C % 64 != 0", "to_hl C > 512"]
            + [f"f32_to_plane {k}" for k in ("f16", "bf16", "NCHW", "NHWC", "cp > C", "several channel tiles",
                                              "edge values")]
            + [f"stem pad ({a},{b})" for a in range(3) for b in range(3)]
            + [f"stem cout {c}" for c in (1, 8, 24, 32, 40, 63, 64)]
            + ["stem ragged grid", "stem one-pixel output", "stem odd H or W", "stem out_cstride 128",
               "stem swish saturates"]
            + [f"dw k{k} s{s}" for k in (3, 5) for s in (1, 2)]
            + ["dw sums", "dw no sums", "dw in_cstride > C", "dw in_cstride != out_cstride", "dw out_cstride > C",
               "dw pad_t != pad_l", "dw Ho or Wo 1", "dw ragged tiles"]
            + ["se last chunk 64", "se last chunk 128", "se 1 chunks", "se 2 chunks", "se 3 chunks",
               "se sums_stride > C", "se C % 64 != 0", "se images 1", "se images 73", "se C 8", "se C 65", "se C 4096",
               "se R 1", "se R 1024", "se gate output, one-row projection"]
            + ["f32_to_hilo NCHW", "f32_to_hilo NHWC", "f32_to_hilo cp > C", "f32_to_hilo ragged tiles",
               "f32_to_hilo edge values", "hilo_to_f32", "hilo_to_f32 window", "spatial_sum",
               "spatial_sum ragged chunk", "spatial_sum small terms after a large one"]
            + ["pool_bias temporal", "pool_bias temporal T 1", "pool_bias n_const", "pool_bias n_const = C - 1",
               "pool_bias bias", "pool_bias bias NULL", "pool_bias accumulate", "pool_bias 4 row slices",
               "pool_bias R 1", "pool_bias C 1", "pool_bias CO % 4 != 0"]
            + ["small_linear bias", "small_linear bias NULL", "small_linear accumulate", "small_linear co > 128",
               "small_linear ci 1024"]
            + ["upsample skip", "upsample no skip", "upsample window 8 mod 16", "upsample skip window 8 mod 16",
               "upsample h or w 1", "upsample C 8"])


def test_every_entry_point_and_feature_is_replayed():
    rows = [r for name in SOURCES for r in run_source(name)]
    counts = {f: sum(f in r["features"] for r in rows) for f in REQUIRED}
    print("\nfeature: launches")
    for f in REQUIRED:
        print(f"  {f:<34s} {counts[f]}")
    print("worst error per entry point (fp32 ulps of the terms' magnitudes; se weights: of the exact bound), bar")
    for m in BARS:
        errs = [(r["res"]["errs"][m], r["tag"], BARS[m] * r["res"].get("bar scale", 1.0)) for r in rows
                if m in r["res"]["errs"]]
        if errs:
            e, tag, bar = max(errs)
            print(f"  {m:<14s} {e:10.3g}  bar {bar:<6.3g} over {len(errs):4d} launches, worst: {tag[:70]}")
    assert all(counts.values()), [f for f, c in counts.items() if not c]
