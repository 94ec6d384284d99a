"""GPU: every launch of the prediction stage's per-pixel kernels (stp3_gru_gates, stp3_gru_update,
stp3_channel_norm_act, stp3_dw_ln, stp3_trust_mix, stp3_maxpool2_pad, stp3_hl_copy, stp3_hl_broadcast) against the
float64 reference of their contract (tests/predict_reference.py), and a probe that the Prediction model reads no memory
it has not written.

The launches are recorded from the model -- the eight dense wrappers replaced while it runs, each call's input buffers
cloned and the windows production wrote cloned too: STP3.forward_features of the Prediction model with the nuScenes and
the CARLA gate sets at a 40 x 56 BEV, B = 2, and STP3._predict_hl on (1, 3, 64, 200, 200) present states -- and built
synthetically for what the model never passes: C in {8, 16, 24, 32, 96, 136, 200, 256} (every lane count L of the
three reducing kernels, with and without idle lanes), stp3_dw_ln with k in {1, 3, 15} on 1 x 1, 1 x W and H x 1 maps,
stp3_trust_mix with 1, 2 and 4 destinations, stp3_hl_broadcast over 3 frames with a row stride wider than C,
stp3_maxpool2_pad on one-row and one-column maps, and hostile inputs: trusting-gate logits hundreds apart (a softmax
without its max subtraction overflows), LayerNorm inputs of mean 1e3 and spread 1e-2 (a one-pass variance loses every
digit), saturated gates.

Each launch is replayed twice into fresh buffers: every channel and frame outside the windows the call reads holds the
bf16 NaN 0x7FA5 in both planes, every output buffer is pre-filled with it.  A call whose output buffer is one of its
input buffers (stp3_gru_update with out = h, stp3_channel_norm_act with out = x, the GRU gates into the cell's own
buffer) is replayed a third time that way, in place.  Checked per replay:
  - the written values against the fp64 reference, in fp32 ulps of the magnitudes of each value's terms beyond the
    2^-17 of the hi/lo split, with the bars of BARS; stp3_maxpool2_pad and stp3_hl_copy bitwise, stp3_hl_broadcast
    bitwise the split stp3_f32_to_hilo stores for the same fp32 vector;
  - every stored hi/lo pair a valid split, and no output element left at the sentinel;
  - every element outside the written windows unchanged;
  - the replays bitwise equal to each other, to what production wrote, and the in-place replay to the out-of-place one.
The coverage test asserts that the recorded sources reached every entry point, that the synthetic and recorded launches
reached every L of the three reducing kernels and every listed feature, and prints the worst error per entry point."""
import inspect
import itertools
import time
from dataclasses import dataclass, field
from typing import Optional

import pytest
import torch

from stp3_b200 import dense
from tests import aux_reference as AR
from tests import predict_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT16 = 0x7FA5            # bf16 NaN: every element a call must not read, and every output before a replay
SPLIT = 2.0 ** -17         # what the hi/lo split of a stored value may lose
ULP = 2.0 ** -24

# Bars in fp32 ulps of the magnitudes of each value's terms (tests/predict_reference.py), about 4x the worst measured
# over every launch of this file on an H100 80GB HBM3 (700 W power limit; table in DESIGN.md section 4).
BARS = {"gru_gates": 6, "gru_update": 7, "channel_norm_act": 8, "dw_ln": 8, "trust_mix": 4}

NAMES = ("gru_gates", "gru_update", "channel_norm_act", "dw_ln", "trust_mix", "maxpool2_pad", "hl_copy", "hl_broadcast")
ORIG = {nm: getattr(dense, nm) for nm in NAMES}
# the slot arguments each wrapper reads and writes
IO = {"gru_gates": (("r", "h"), ("out",)), "gru_update": (("u", "h", "h_tilde"), ("out", "out2")),
      "channel_norm_act": (("x", "y"), ("out",)), "dw_ln": (("x",), ("out",)), "trust_mix": (("t", "s1", "s2"), ("dsts",)),
      "maxpool2_pad": (("x",), ("out",)), "hl_copy": (("src",), ("dst",)), "hl_broadcast": ((), ("dst",))}
REDUCING = ("channel_norm_act", "dw_ln", "trust_mix")


def lanes(C):
    """lanes per pixel of the reducing kernels (csrc/predict_kernels.cu lanes_for)"""
    L = 1
    while L * 8 < C:
        L *= 2
    return L


def _bits(t):
    return t.contiguous().view(torch.int16)


def _is_sent(t):
    return _bits(t) == SENT16


def _sent_like(shape):
    return torch.full(shape, SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _slot(v):
    """(HL, coff, t0) of a slot argument"""
    return (v + (0, 0))[:3] if isinstance(v, tuple) else (v, 0, 0)


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    kind: str
    bufs: list                  # per buffer: (hi, lo) cloned input planes, or None for an output-only buffer
    shapes: list                # per buffer: (B, T_total, H, W, cstride)
    ins: dict                   # role -> (buffer, coff, t0)
    outs: dict                  # role -> (buffer, coff, t0)
    C: int
    T: int
    p: dict                     # parameters
    tag: str = ""
    prod: Optional[dict] = None  # role -> (hi, lo) window production wrote
    features: set = field(default_factory=set)

    def window(self, role):
        b, coff, t0 = {**self.ins, **self.outs}[role]
        C = self.shapes[b][-1] if self.kind == "maxpool2_pad" else self.C
        return (slice(None), slice(t0, t0 + self.T), slice(None), slice(None), slice(coff, coff + C))

    @property
    def aliased(self):
        return any(b in {i for i, _, _ in self.ins.values()} for b, _, _ in self.outs.values())


def _features(c: Case) -> set:
    k, C, p = c.kind, c.C, c.p
    f = {k}
    if k in REDUCING:
        L = lanes(C)
        f.add(f"{k} L{L}")
        if C < 8 * L:
            f.add(f"{k} L{L} idle lanes")
    if any(coff for _, coff, _ in list(c.ins.values()) + list(c.outs.values())):
        f.add("slot coff > 0")
    if any(t0 for _, _, t0 in list(c.ins.values()) + list(c.outs.values())):
        f.add("frame slot t0 > 0")
    if c.aliased:
        f.add(f"{k} in place")
    _, _, H, W, _ = c.shapes[next(iter(c.ins.values()))[0] if c.ins else next(iter(c.outs.values()))[0]]
    if k == "dw_ln":
        f.add(f"dw_ln k{p['k']}")
        if H < p["k"] or W < p["k"]:
            f.add("dw_ln map smaller than the window")
        if H == 1 and W == 1:
            f.add("dw_ln 1x1 map")
        elif H == 1:
            f.add("dw_ln 1xW map")
        elif W == 1:
            f.add("dw_ln Hx1 map")
    if k == "trust_mix":
        f.add(f"trust_mix {len(c.outs)} destinations")
    if k == "channel_norm_act":
        f.add("channel_norm_act LN" if p["ln"] is not None else "channel_norm_act no LN")
        if "y" in c.ins:
            f.add("channel_norm_act gelu(y)" if p["gelu_y"] else "channel_norm_act y")
    if k == "gru_update" and "out2" in c.outs:
        f.add("gru_update out2")
    if k == "hl_broadcast":
        if c.T > 1:
            f.add("hl_broadcast T > 1")
        if p["vec"].shape[1] > C:
            f.add("hl_broadcast vstride > C")
    if k == "maxpool2_pad":
        f |= {nm for nm, on in (("maxpool2_pad odd H", H % 2), ("maxpool2_pad odd W", W % 2),
                                ("maxpool2_pad 1-row map", H == 1), ("maxpool2_pad 1-column map", W == 1)) if on}
    return f


# ------------------------------------------------------------------------------------------------ recording
class Recorder:
    """Replaces the eight dense wrappers while the model runs; every call becomes a Case with clones of its input
    buffers and of the windows production wrote."""

    def __init__(self, source):
        self.source, self.cases = source, []

    def __enter__(self):
        self.mp = pytest.MonkeyPatch()
        for nm in NAMES:
            self.mp.setattr(dense, nm, self._wrap(nm))
        return self

    def __exit__(self, *exc):
        self.mp.undo()
        torch.cuda.synchronize()

    def _wrap(self, nm):
        orig, sig = ORIG[nm], inspect.signature(ORIG[nm])
        in_roles, out_roles = IO[nm]

        def f(*args, **kw):
            a = sig.bind(*args, **kw)
            a.apply_defaults()
            a = dict(a.arguments)
            bufs, shapes, ptrs = [], [], {}

            def buf(hl, clone):
                i = ptrs.get(hl.hi.data_ptr())
                if i is None:
                    i = ptrs[hl.hi.data_ptr()] = len(bufs)
                    bufs.append((hl.hi.clone(), hl.lo.clone()) if clone else None)
                    shapes.append(tuple(hl.hi.shape))
                return i
            ins = {}
            for r in in_roles:
                if a.get(r) is not None:
                    hl, coff, t0 = _slot(a[r])
                    ins[r] = (buf(hl, True), coff, t0)
            outs = {}
            dst = a.get("dsts") if nm == "trust_mix" else None
            pending = [(f"d{i}", d) for i, d in enumerate(dst)] if dst is not None else \
                [(r, a[r]) for r in out_roles if a.get(r) is not None]
            ret = orig(*args, **kw)
            if nm == "maxpool2_pad" and a["out"] is None:
                pending = [("out", ret)]
            for r, v in pending:
                hl, coff, t0 = _slot(v)
                outs[r] = (buf(hl, False), coff, t0)
            x0 = _slot(a[in_roles[0]] if in_roles else a["dst"])
            C = a["x"].hi.shape[-1] if nm == "maxpool2_pad" else a["C"]
            T = a.get("T")
            if T is None:
                T = x0[0].hi.shape[1] - x0[2]
            p = {k: v for k, v in a.items() if k not in in_roles + out_roles + ("C", "T")}
            p = {k: (v.clone() if torch.is_tensor(v) else tuple(t.clone() if torch.is_tensor(t) else t for t in v)
                     if isinstance(v, tuple) else v) for k, v in p.items()}
            c = Case(nm, bufs, shapes, ins, outs, C, T, p, tag=f"{self.source}: {nm} C{C} T{T} {shapes[0][2:4]}")
            c.prod = {}
            for r, v in pending:
                hl, w = _slot(v)[0], c.window(r)
                c.prod[r] = (hl.hi[w].clone(), hl.lo[w].clone())
            c.features = _features(c) | {"recorded", f"recorded {nm}"}
            self.cases.append(c)
            return ret
        return f


# ------------------------------------------------------------------------------------------------ replay
def _materialise(c: Case, in_place: bool):
    """{role: (HL, coff, t0)} of fresh buffers: inputs NaN outside the windows the call reads; outputs sentinel, or in
    place the input buffer they share"""
    read = {}
    for r, (b, _, _) in c.ins.items():
        m = read.setdefault(b, torch.zeros(c.shapes[b][1], c.shapes[b][4], dtype=torch.bool, device=DEV))
        w = c.window(r)
        m[w[1], w[4]] = True
    hls = {}
    for b, m in read.items():
        hi, lo = c.bufs[b]
        m5 = m.view(1, m.shape[0], 1, 1, m.shape[1])
        hls[b] = dense.HL(torch.where(m5, hi, _sent_like(hi.shape)), torch.where(m5, lo, _sent_like(lo.shape)),
                          c.shapes[b][-1])
    slots = {r: (hls[b], coff, t0) for r, (b, coff, t0) in c.ins.items()}
    fresh = {}
    for r, (b, coff, t0) in c.outs.items():
        if in_place and b in hls:
            hl = hls[b]
        else:
            if b not in fresh:
                fresh[b] = dense.HL(_sent_like(c.shapes[b]), _sent_like(c.shapes[b]), c.shapes[b][-1])
            hl = fresh[b]
        slots[r] = (hl, coff, t0)
    before = {r: (s[0].hi.clone(), s[0].lo.clone()) for r, s in slots.items() if r in c.outs}
    return slots, before


def _launch(c: Case, s: dict):
    k, p, C, T = c.kind, c.p, c.C, c.T
    if k == "gru_gates":
        ORIG[k](s["r"], s["h"], s["out"], C, T=T)
    elif k == "gru_update":
        ORIG[k](s["u"], s["h"], s["h_tilde"], s["out"], C, out2=s.get("out2"), T=T)
    elif k == "channel_norm_act":
        ORIG[k](s["x"], s["out"], C, ln=p["ln"], gelu=p["gelu"], y=s.get("y"), gelu_y=p["gelu_y"], T=T)
    elif k == "dw_ln":
        ORIG[k](s["x"], p["w"], p["b"], p["k"], p["ln"], s["out"], C, T=T)
    elif k == "trust_mix":
        ORIG[k](s["t"], p["w"], s["s1"], s["s2"], [s[f"d{i}"] for i in range(len(c.outs))], C, T=T)
    elif k == "maxpool2_pad":
        ORIG[k](s["x"][0], out=s["out"][0])
    elif k == "hl_copy":
        ORIG[k](s["src"], s["dst"], C, T=T)
    elif k == "hl_broadcast":
        ORIG[k](p["vec"], s["dst"], C, T=T)
    else:
        raise AssertionError(k)


def replay(c: Case, in_place: bool):
    """-> ({role: (hi, lo) written window}, {role: nothing outside the window changed})"""
    slots, before = _materialise(c, in_place)
    _launch(c, slots)
    torch.cuda.synchronize()
    got, untouched = {}, {}
    for r in c.outs:
        hl = slots[r][0]
        w = c.window(r)
        got[r] = (hl.hi[w].clone(), hl.lo[w].clone())
        keep = torch.ones(hl.hi.shape, dtype=torch.bool, device=DEV)
        keep[w] = False
        for rr in c.outs:                     # other destinations in the same buffer
            if slots[rr][0] is hl:
                keep[c.window(rr)] = False
        untouched[r] = bool(torch.equal(_bits(hl.hi)[keep], _bits(before[r][0])[keep]) and
                            torch.equal(_bits(hl.lo)[keep], _bits(before[r][1])[keep]))
    return got, untouched


# ------------------------------------------------------------------------------------------------ checks
def _val(c: Case, role):
    b = {**c.ins}[role][0]
    hi, lo = c.bufs[b]
    w = c.window(role)
    return R.planes(hi[w], lo[w])


def reference(c: Case) -> dict:
    """{"y": value of every written element (B, T, H, W, C), "mag": its magnitude} or {"hi", "lo"} for bitwise kinds"""
    k, p = c.kind, c.p
    if k == "gru_gates":
        return R.gru_gates(_val(c, "r"), _val(c, "h"))
    if k == "gru_update":
        return R.gru_update(_val(c, "u"), _val(c, "h"), _val(c, "h_tilde"))
    if k == "channel_norm_act":
        return R.channel_norm_act(_val(c, "x"), p["ln"], p["gelu"], _val(c, "y") if "y" in c.ins else None, p["gelu_y"])
    if k == "dw_ln":
        x = _val(c, "x")
        B, T, H, W, C = x.shape
        r = R.dw_ln(x.reshape(B * T, H, W, C), p["w"], p["b"], p["k"], *p["ln"])
        return {n: v.reshape(B, T, H, W, C) for n, v in r.items()}
    if k == "trust_mix":
        return R.trust_mix(_val(c, "t"), p["w"], _val(c, "s1"), _val(c, "s2"))
    if k == "maxpool2_pad":
        hi, lo = c.bufs[c.ins["x"][0]]
        B, T, H, W, cs = hi.shape
        oh, ol = R.maxpool2_pad(hi.reshape(B * T, H, W, cs), lo.reshape(B * T, H, W, cs))
        return {"hi": oh.reshape(B, T, *oh.shape[1:]), "lo": ol.reshape(B, T, *ol.shape[1:])}
    if k == "hl_copy":
        hi, lo = c.bufs[c.ins["src"][0]]
        w = c.window("src")
        return {"hi": hi[w], "lo": lo[w]}
    if k == "hl_broadcast":
        B, _, H, W, _ = c.shapes[c.outs["dst"][0]]
        hi, lo = AR.split(p["vec"][:, :c.C])
        ex = lambda t: t.view(B, c.T, 1, 1, c.C).expand(B, c.T, H, W, c.C)     # noqa: E731
        return {"hi": ex(hi), "lo": ex(lo)}
    raise AssertionError(k)


def _excess(hi, lo, ref, mag):
    """max over elements of the planes' error beyond the split allowance, in fp32 ulps of mag (NaN if any is NaN)"""
    e = ((R.planes(hi, lo) - ref).abs() - SPLIT * ref.abs()).clamp_min(0)
    return float((e / (ULP * mag + 1e-300)).max()) if e.numel() else 0.0


def _same(a, b):
    return all(torch.equal(_bits(a[r][0]), _bits(b[r][0])) and torch.equal(_bits(a[r][1]), _bits(b[r][1])) for r in a)


def check(c: Case) -> dict:
    """-> {"errs": {metric: error}, flag: bool, ...}; asserts nothing"""
    g1, u1 = replay(c, False)
    g2, u2 = replay(c, False)
    res = {"untouched": all(u1.values()) and all(u2.values()), "same": _same(g1, g2)}
    if c.aliased:
        g3, u3 = replay(c, True)
        res["in place untouched"] = all(u3.values())
        res["in place same"] = _same(g1, g3)
    if c.prod is not None:
        res["production"] = _same(c.prod, g1)
    res["written"] = not any(bool((_is_sent(hi) & _is_sent(lo)).any()) for hi, lo in g1.values())
    res["split"] = all(bool(AR.split_valid(hi, lo).all()) for hi, lo in g1.values())
    ref = reference(c)
    errs = {}
    if "y" in ref:
        errs[c.kind] = max(_excess(hi, lo, ref["y"], ref["mag"]) for hi, lo in g1.values())
    else:
        res["bitwise"] = all(torch.equal(_bits(hi), _bits(ref["hi"])) and torch.equal(_bits(lo), _bits(ref["lo"]))
                             for hi, lo in g1.values())
    if "hostile softmax" in c.features:
        res["saturated"] = bool(((ref["p"] < 1e-30) | (ref["p"] > 1 - 1e-15)).any())
    res["errs"] = errs
    return res


def passed(res):
    return all(v for v in res.values() if isinstance(v, bool)) and all(e <= BARS[m] for m, e in res["errs"].items())


# ------------------------------------------------------------------------------------------------ synthetic launches
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def rand_hl(B, T, H, W, cs, seed, scale=1.0, offset=0.0):
    x = torch.randn((B, T, H, W, cs), generator=_gen(seed), device=DEV) * scale + offset
    hi, lo = AR.split(x)
    return dense.HL(hi.contiguous(), lo.contiguous(), cs)


def rnd(*shape, seed, scale=1.0, offset=0.0):
    return torch.randn(shape, generator=_gen(seed), device=DEV) * scale + offset


def _ln(C, seed):
    return (rnd(C, seed=seed, scale=0.5, offset=1.0), rnd(C, seed=seed + 1, scale=0.2), 1e-6)


def synthetic(hostile=False):
    """launches the model never makes; recorded through the same wrappers (the Recorder clones what they wrote)"""
    s = [0]

    def sd():
        s[0] += 1
        return 5000 + s[0]
    B, T = 2, 2
    Cs = (8, 16, 24, 32, 96, 136, 200, 256)
    if not hostile:
        for C in Cs:
            cs = C + 16
            H, W = 5, 7
            x, y = rand_hl(B, T + 1, H, W, cs, sd()), rand_hl(B, T, H, W, cs, sd())
            dense.channel_norm_act((x, 8, 1), (dense.HL.empty(B, T, H, W, cs, DEV, cp=cs), 8), C, ln=_ln(C, sd()),
                                   gelu=True, y=(y, 16), gelu_y=C % 16 == 0, T=T)
            x2 = rand_hl(B, T, H, W, C, sd())
            dense.channel_norm_act(x2, x2, C, ln=_ln(C, sd()))                        # in place
            dense.channel_norm_act((x, 0, 1), dense.HL.empty(B, T, H, W, C, DEV, cp=C), C, gelu=True, T=T)
            k = 3 if C < 100 else 7
            dense.dw_ln((x, 8), rnd(k * k, C, seed=sd(), scale=1.0 / k), rnd(C, seed=sd(), scale=0.1), k, _ln(C, sd()),
                        (dense.HL.empty(B, T + 1, H, W, cs, DEV, cp=cs), 16), C)
            t, s12 = rand_hl(B, T, H, W, C, sd()), rand_hl(B, T, H, W, 2 * C, sd())
            dense.trust_mix(t, rnd(2, C, seed=sd(), scale=C ** -0.5), (s12, 0), (s12, C),
                            [dense.HL.empty(B, T, H, W, C, DEV, cp=C)], C)
        for k, (H, W) in itertools.product((1, 3, 15), ((1, 1), (1, 9), (9, 1), (4, 6))):
            C = 24 if k != 15 else 136
            x = rand_hl(B, T, H, W, C, sd())
            dense.dw_ln(x, rnd(k * k, C, seed=sd(), scale=1.0 / k), rnd(C, seed=sd(), scale=0.1), k, _ln(C, sd()),
                        dense.HL.empty(B, T, H, W, C, DEV, cp=C), C)
        for n_dst in (1, 2, 4):
            C, H, W = 64, 6, 9
            t, s1, s2 = (rand_hl(B, T, H, W, C, sd()) for _ in range(3))
            out = dense.HL.empty(B, T + 2, H, W, 128, DEV, cp=128)
            dsts = [(out, 64 * (i % 2), 2 * (i // 2)) for i in range(n_dst)]
            dense.trust_mix(t, rnd(2, C, seed=sd(), scale=0.1), s1, s2, dsts, C, T=T)
        vec = rnd(B * 3, 72, seed=sd())
        dense.hl_broadcast(vec, (dense.HL.empty(B, 5, 4, 7, 64, DEV, cp=64), 16, 1), 40, T=3)
        for H, W in ((1, 9), (9, 1), (1, 1), (7, 8)):
            dense.maxpool2_pad(rand_hl(B, T, H, W, 64, sd()))
        g, h, ht = rand_hl(B, T, 3, 5, 128, sd(), 3.0), rand_hl(B, T, 3, 5, 64, sd()), rand_hl(B, T, 3, 5, 64, sd())
        dense.gru_gates((g, 64), h, (dense.HL.empty(B, T + 1, 3, 5, 192, DEV, cp=192), 128, 1), 64, T=T)
        dense.gru_update(g, h, ht, h, 64, out2=(dense.HL.empty(B, T, 3, 5, 64, DEV, cp=64), 0))
        dense.hl_copy((h, 8), (dense.HL.empty(B, T + 1, 3, 5, 64, DEV, cp=64), 16, 1), 40, T=T)
        return
    # hostile inputs
    C, H, W = 64, 5, 6
    t = rand_hl(B, T, H, W, C, sd(), scale=40.0)                       # logits ~ +-300: exp(z) overflows fp32
    s1, s2 = rand_hl(B, T, H, W, C, sd()), rand_hl(B, T, H, W, C, sd())
    dense.trust_mix(t, rnd(2, C, seed=sd()), s1, s2, [dense.HL.empty(B, T, H, W, C, DEV, cp=C)], C)
    for C in (24, 64, 200):
        x = rand_hl(B, T, H, W, C, sd(), scale=1e-2, offset=1e3)      # mean 1e3, spread 1e-2
        dense.channel_norm_act(x, dense.HL.empty(B, T, H, W, C, DEV, cp=C), C, ln=_ln(C, sd()), gelu=True)
        x = rand_hl(B, T, H, W, C, sd(), scale=3e-3)                  # depthwise output 1e3 + 1e-2 noise
        dense.dw_ln(x, rnd(9, C, seed=sd()), rnd(C, seed=sd(), scale=0.0, offset=1e3), 3, _ln(C, sd()),
                    dense.HL.empty(B, T, H, W, C, DEV, cp=C), C)
    g, h, ht = rand_hl(B, T, H, W, 128, sd(), 60.0), rand_hl(B, T, H, W, 64, sd()), rand_hl(B, T, H, W, 64, sd())
    dense.gru_gates((g, 64), h, dense.HL.empty(B, T, H, W, 64, DEV, cp=64), 64)
    dense.gru_update(g, h, ht, dense.HL.empty(B, T, H, W, 64, DEV, cp=64), 64)


def rec_synthetic(hostile):
    with Recorder("hostile" if hostile else "synthetic") as r:
        synthetic(hostile)
    for c in r.cases:
        if hostile:
            c.features.add({"trust_mix": "hostile softmax", "channel_norm_act": "hostile LayerNorm mean 1e3",
                            "dw_ln": "hostile LayerNorm mean 1e3"}.get(c.kind, "saturated gates"))
        c.features -= {"recorded", f"recorded {c.kind}"}
    return r.cases


def rec_predict_small(carla):
    from tests import test_conv_contract_gpu as CC
    r = Recorder(f"predict {'carla' if carla else 'nuscenes'} 40x56")
    CC.run_predict_small(carla, r)
    return r.cases


def rec_predict_200():
    from tests import test_conv_contract_gpu as CC
    r = Recorder("predict 200x200")
    CC.run_predict_200(r)
    return r.cases


SOURCES = {
    "predict_small_nuscenes": lambda: rec_predict_small(False),
    "predict_small_carla": lambda: rec_predict_small(True),
    "predict_200x200": rec_predict_200,
    "synthetic": lambda: rec_synthetic(False),
    "hostile": lambda: rec_synthetic(True),
}
_RUNS = {}


def run_source(name):
    if name in _RUNS:
        return _RUNS[name]
    t0 = time.time()
    cases = SOURCES[name]()
    assert cases, f"{name}: no launch recorded"
    rows = []
    for c in cases:
        r = check(c)
        rows.append(dict(kind=c.kind, tag=c.tag, features=set(c.features), res=r, ok=passed(r)))
    del cases
    torch.cuda.empty_cache()
    print(f"\n{name}: {len(rows)} launches in {time.time() - t0:.1f} s")
    _RUNS[name] = rows
    return rows


def _fmt(r):
    res = r["res"]
    s = " ".join(f"{m} {e:.3g}" for m, e in res["errs"].items())
    flags = [k for k, v in res.items() if isinstance(v, bool) and not v]
    return f"  {r['kind']:<16s} {r['tag'][:76]:<76s} {s}" + (f"  FAILED {flags}" if flags else "")


@pytest.mark.parametrize("name", list(SOURCES))
def test_predict_launches_against_the_fp64_contract(name):
    rows = run_source(name)
    for r in rows:
        print(_fmt(r))
    bad = [_fmt(r) for r in rows if not r["ok"]]
    assert not bad, "\n".join(bad)


REQUIRED = ([f"recorded {k}" for k in NAMES]
            + [f"{k} L{L}" for k in REDUCING for L in (1, 2, 4, 8, 16, 32)]
            + [f"{k} L{L} idle lanes" for k in REDUCING for L in (4, 32)]
            + [f"dw_ln k{k}" for k in (1, 3, 7, 15)]
            + ["dw_ln map smaller than the window", "dw_ln 1x1 map", "dw_ln 1xW map", "dw_ln Hx1 map"]
            + [f"trust_mix {n} destinations" for n in (1, 2, 3, 4)]
            + ["hl_broadcast T > 1", "hl_broadcast vstride > C", "maxpool2_pad odd H", "maxpool2_pad odd W",
               "maxpool2_pad 1-row map", "maxpool2_pad 1-column map", "gru_update in place",
               "channel_norm_act in place", "gru_update out2", "channel_norm_act LN", "channel_norm_act no LN",
               "channel_norm_act y", "channel_norm_act gelu(y)", "slot coff > 0", "frame slot t0 > 0",
               "hostile softmax", "hostile LayerNorm mean 1e3", "saturated gates"])


def test_every_entry_point_lane_count_and_feature_is_replayed():
    rows = [r for name in SOURCES for r in run_source(name)]
    counts = {f: sum(f in r["features"] for r in rows) for f in REQUIRED}
    print("\nfeature: launches")
    for f in REQUIRED:
        print(f"  {f:<36s} {counts[f]}")
    print("worst error per entry point (fp32 ulps of the terms' magnitudes beyond 2^-17), bar")
    for m in BARS:
        errs = [(r["res"]["errs"][m], r["tag"]) for r in rows if m in r["res"]["errs"]]
        if errs:
            e, tag = max(errs)
            print(f"  {m:<18s} {e:10.3g}  bar {BARS[m]:<4g} over {len(errs):4d} launches, worst: {tag[:70]}")
    for k in NAMES:
        if k not in BARS:
            print(f"  {k:<18s}    bitwise  over {sum(r['kind'] == k for r in rows):4d} launches")
    assert all(counts.values()), [f for f, c in counts.items() if not c]


# ------------------------------------------------------------------------------------------------ unwritten memory
@pytest.mark.parametrize("carla", [False, True], ids=["nuscenes", "carla"])
def test_prediction_model_reads_no_unwritten_memory(carla, monkeypatch):
    """predict_small_* under torch.use_deterministic_algorithms, once with every dense.HL.empty buffer zero-filled and
    once with it bf16 NaN in both planes: every output finite and bitwise equal between the two runs.  A launch whose
    reads cover an element nobody wrote (a zero-weight K range, a padding channel) multiplies NaN by zero; the NaN need
    not reach the outputs -- a ReLU epilogue (fmaxf) turns it into 0 -- but the values it passes on differ from the
    zero-filled run's.  (The comparison is against zero-filled buffers, not as-is ones: in deterministic mode torch
    fills uninitialised memory with NaN itself.)"""
    from tests import test_conv_contract_gpu as CC
    from contextlib import nullcontext

    def filled(bits):
        def empty(B, T, H, W, c, device, cp=None):
            cp = cp or dense.pad_to(c)
            plane = lambda: torch.full((B, T, H, W, cp), bits, dtype=torch.int16, device=device).view(torch.bfloat16)  # noqa: E731
            return dense.HL(plane(), plane(), c)
        return staticmethod(empty)
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for bits in (0, 0x7FC0):
            monkeypatch.setattr(dense.HL, "empty", filled(bits))
            out = CC.run_predict_small(carla, nullcontext())
            runs.append({k: v.clone() for k, v in out.items() if torch.is_tensor(v)})
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    a, b = runs
    assert set(a) == set(b) and a
    for k in a:
        print(f"  {k:20s} {tuple(a[k].shape)} finite {bool(torch.isfinite(b[k]).all())} "
              f"bitwise {torch.equal(a[k], b[k])}")
        assert bool(torch.isfinite(a[k]).all()) and bool(torch.isfinite(b[k]).all()), k
        assert torch.equal(a[k], b[k]), k
