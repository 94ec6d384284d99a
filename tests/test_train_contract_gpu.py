"""GPU: every train-mode launch of stp3_b200/csrc/train_kernels.cu against the float64 reference of its contract
(tests/train_reference.py).

The launches come from full train steps of the models (the dense_train functions wrapped while a forward and backward
run: the decoder with all gates at 48 x 64 and at 200 x 200, the DeepLab head, the TemporalModel, the encoder heads, the
trainable EfficientNet trunk: b0 and b4 on 3 x 35 x 51 images and b4 on 6 x 224 x 480, trunk_step) and
from synthetic calls through _lib.lib() for what the wrappers never produce: wide and odd row strides, pointers off
16-byte alignment (the scalar paths), channel counts from 1 to 1030, maps of one row or column, stride 2, dilations
whose taps lie partly or wholly in the padding, dead time taps, empty trailing K splits, dropout offsets past 2^32.
Each launch is replayed twice into outputs filled with a sentinel (the whole wide tensor of a windowed output, the bf16
planes with their padding), inputs placed in NaN-filled rows (a read outside the window shows) and scratch filled with
0xFF bytes (NaN: scratch has no invariant).  Checked per launch:
  - the weight gradient against the exact fp64 product (of max |exact|) and, element by element, its excess over the
    fp64 evaluation of the three bf16 products the kernel issues, with a bar measured on the H100 (wgrad_bar);
  - the elementwise kernels within a few fp32 ulps of the summed magnitudes of their terms, the fp64-accumulated
    reductions within one rounding of the result plus the fp32 rounding of their terms;
  - nothing outside the written window changed; bf16 padding channels exactly zero; the bf16 planes bitwise the
    hi/lo split of the stored fp32 output; the dropout mask bit for bit the header's Philox-4x32-10; g_masked bitwise
    where(y > 0, g, 0); phase_interleave an exact copy;
  - the two replays bitwise equal, and equal to what the production launch wrote.
One-plane (autocast) launches: the same modules run steps with the forward under torch.autocast in float16 and in
bfloat16 (one of them at 200 x 200, so the weight gradient's pixels per split reach the thousands), and synthetic calls
cover what they never produce.  stp3_conv_wgrad_plane / stp3_conv3d_wgrad_plane are replayed on the plane bytes
production read (the forward's kept plane or the operand() plane, at its row stride; an fp32 operand as the plane
stp3_f32_to_plane makes of it, torch's rounding, which tests/test_aux_contract_gpu.py holds it to bit for bit), in rows
whose channels outside [0, cin) are a NaN of the plane type, and held to the fp64 product of the plane values within
wgrad_bar(per) of its max; stp3_bn_apply_plane must store y bitwise as stp3_bn_apply does on the same arguments, the
plane bitwise torch's rounding of y with padding channels +0, and the dropout bits of the Philox reference.
The last test asserts that the replays reached every entry point and path."""
import ast
import inspect
import os
import time
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pytest
import torch

from oracle import torch_dense as TD
from stp3_b200 import _lib, dense, dense_train
from tests import train_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -1.5e30
ULP = 2.0 ** -24


# Weight gradient bars, of max |exact| over the output.  The kernel's only departures from the three-product model are
# its fp32 sums: one 64-pixel stage chained in the tensor cores, then per / 64 stage sums added in fp32 (round to
# nearest), so the excess grows like sqrt(per), per = the output pixels of one K split (tests/train_reference.py
# wgrad_split).  Worst measured on an H100 80GB HBM3 (700 W power limit) over every recorded and synthetic launch (table
# in DESIGN.md section 3.10): 4.2e-7 at per = 64, 8.8e-7 at 256, 1.8e-6 at 960, 3.1e-6 at 7296, 2.3e-6 at 8000, all
# below 2e-7 + 6e-8 sqrt(per).  The bar is 4x that envelope.  Dropping one of the three products moves a random-data
# gradient by ~2^-9 / sqrt(3) of its inputs' scale, far above it at every per.
def wgrad_bar(per: int) -> float:
    return 4 * (2e-7 + 6e-8 * per ** 0.5)


# Against the exact product the bf16 x 3 representation (no lo x lo term, 2^-16 relative per product) dominates: worst
# measured 4.0e-5 for a 1x1 over six one-pixel images, where the sum cancels, and <= 9e-6 everywhere else.  Sums of
# fewer than 64 products may cancel further (the trunk's squeeze-excite weights: 1.56e-4 of max over six images), so
# there the bar also accepts 1e-4 of the representation bound 2^-16 sum |x g| (check)
WGRAD_EXACT_BAR = 1e-4


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ buffers
@dataclass
class In:
    """An fp32 input of n rows x C channels at row stride cs, window starting at column coff, the storage shifted by
    `shift` elements (shift % 4 != 0: not 16-byte aligned); every element outside the window is NaN."""
    vals: torch.Tensor                 # (n, C) fp32
    cs: int = 0
    coff: int = 0
    shift: int = 0

    def __post_init__(self):
        self.vals = self.vals.detach().reshape(-1, self.vals.shape[-1]).float().to(DEV).clone()
        n, C = self.vals.shape
        self.cs = self.cs or C
        self.store = torch.full((self.shift + n * self.cs + 16,), float("nan"), device=DEV)
        self.store[self.shift:self.shift + n * self.cs].view(n, self.cs)[:, self.coff:self.coff + C] = self.vals

    def ptr(self):
        return self.store.data_ptr() + 4 * (self.shift + self.coff)

    def aligned(self):
        return self.cs % 4 == 0 and (self.shift + self.coff) % 4 == 0


NAN16 = 0x7FFF          # a NaN of both fp16 and bf16
SENT16 = 0x7FA5         # sentinel of one-plane outputs (also a NaN of both types)


@dataclass
class PIn:
    """A one-plane (fp16 / bf16) input of n rows x C channels at row stride cs, the storage shifted by `shift` elements
    (shift % 8 != 0: not 16-byte aligned); every element outside channels [0, C) is NaN of the plane type."""
    vals: torch.Tensor                 # (n, C) fp16 / bf16
    cs: int = 0
    shift: int = 0
    coff = 0

    def __post_init__(self):
        self.vals = self.vals.detach().reshape(-1, self.vals.shape[-1]).to(DEV).clone()
        n, C = self.vals.shape
        self.cs = self.cs or C
        self.store = torch.full((self.shift + n * self.cs + 16,), NAN16, dtype=torch.int16, device=DEV).view(self.vals.dtype)
        self.store[self.shift:self.shift + n * self.cs].view(n, self.cs)[:, :C] = self.vals

    def ptr(self):
        return self.store.data_ptr() + 2 * self.shift

    def aligned(self):
        return self.cs % 8 == 0 and self.shift % 8 == 0


def _plane_operand(t, mode):
    """(plane values (rows, C), row stride, (H, W), (B, T) or None) of what dense_train.conv_wgrad reads under `mode`:
    a one-plane HL as it is, an fp32 tensor as operand() converts it (cp = pad_to(C))"""
    if isinstance(t, dense.HL):
        B, T, H, W, cs = t.hi.shape
        return t.hi.reshape(-1, cs)[:, :t.c], cs, (H, W), None
    C = t.shape[-1]
    return t.reshape(-1, C).to(mode), dense.pad_to(C), tuple(t.shape[-3:-1]), tuple(t.shape[:2]) if t.dim() == 5 else None


def In_of(t: torch.Tensor) -> In:
    """a production tensor (a contiguous one, or a channel window of a wider channels-last one) as an In with the same
    row stride, window offset and 16-byte alignment"""
    cs = t.stride(-2) if t.dim() >= 2 else t.shape[-1]
    coff = t.storage_offset() % cs
    x = In(t.reshape(-1, t.shape[-1]), cs, coff)
    assert (x.ptr() - t.data_ptr()) % 16 == 0
    return x


@dataclass
class Out:
    """An fp32 output window of n rows x C channels at row stride cs from column coff (storage shifted by `shift`)"""
    n: int
    C: int
    cs: int = 0
    coff: int = 0
    shift: int = 0

    def __post_init__(self):
        self.cs = self.cs or self.C

    def alloc(self):
        store = torch.full((self.shift + self.n * self.cs + 16,), SENT, device=DEV)
        keep = torch.ones_like(store, dtype=torch.bool)
        keep[self.shift:self.shift + self.n * self.cs].view(self.n, self.cs)[:, self.coff:self.coff + self.C] = False
        return store, keep

    def window(self, store):
        return store[self.shift:self.shift + self.n * self.cs].view(self.n, self.cs)[:, self.coff:self.coff + self.C]

    def ptr(self, store):
        return store.data_ptr() + 4 * (self.shift + self.coff)

    def aligned(self):
        return self.cs % 4 == 0 and (self.shift + self.coff) % 4 == 0


def _dense_out(shape):
    n = int(np.prod(shape))
    return Out(1, n)


def _scratch(nbytes):
    return torch.full((max(int(nbytes), 1),), 0xFF, dtype=torch.uint8, device=DEV)


def _vec(t):
    return t.detach().float().contiguous().to(DEV).clone()


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    kind: str
    a: dict
    tag: str = ""
    prod: Optional[dict] = None            # what the production launch wrote, per output name
    features: set = field(default_factory=set)


def run(case: Case):
    """Launch the case once into fresh sentinel-filled outputs and 0xFF scratch -> ({name: written values},
    {name: (storage, keep mask)})"""
    L, a, k = _lib.lib(), case.a, case.kind
    outs = {}

    def out(name, spec):
        store, keep = spec.alloc()
        outs[name] = (spec, store, keep)
        return spec.ptr(store)
    if k == "wgrad":
        x, g = a["x"], a["g"]
        shape = (a["cout"], a["cin"], a["kt"], a["kh"], a["kw"])
        dw = out("dw", _dense_out(shape))
        op = dense.PLANE_OPERAND[a["mode"]] if a["mode"] is not None else None
        if op is not None and a["is3d"]:
            nb = L.stp3_conv3d_wgrad_scratch_bytes(a["B"], a["T"], a["H"], a["W"], a["cout"], a["cin"], a["kt"], a["kh"], a["kw"])
            sc = _scratch(nb)
            code = L.stp3_conv3d_wgrad_plane(op, x.ptr(), a["B"], a["T"], a["H"], a["W"], x.cs, a["cin"], g.ptr(), g.cs,
                                             a["cout"], a["kt"], a["kh"], a["kw"], sc.data_ptr(), nb, dw, _stream())
        elif op is not None:
            nb = L.stp3_conv_wgrad_scratch_bytes(a["n_img"], a["Ho"], a["Wo"], a["cout"], a["cin"], a["kh"], a["kw"], a["dil"])
            sc = _scratch(nb)
            code = L.stp3_conv_wgrad_plane(op, x.ptr(), a["n_img"], a["H"], a["W"], x.cs, a["cin"], g.ptr(), a["Ho"],
                                           a["Wo"], g.cs, a["cout"], a["kh"], a["kw"], a["stride"], a["pad"], a["dil"],
                                           sc.data_ptr(), nb, dw, _stream())
        elif a["is3d"]:
            nb = L.stp3_conv3d_wgrad_scratch_bytes(a["B"], a["T"], a["H"], a["W"], a["cout"], a["cin"], a["kt"], a["kh"], a["kw"])
            sc = _scratch(nb)
            code = L.stp3_conv3d_wgrad(x.ptr(), a["B"], a["T"], a["H"], a["W"], x.cs, a["cin"], g.ptr(), g.cs, a["cout"],
                                       a["kt"], a["kh"], a["kw"], sc.data_ptr(), nb, dw, _stream())
        else:
            nb = L.stp3_conv_wgrad_scratch_bytes(a["n_img"], a["Ho"], a["Wo"], a["cout"], a["cin"], a["kh"], a["kw"], a["dil"])
            sc = _scratch(nb)
            code = L.stp3_conv_wgrad(x.ptr(), a["n_img"], a["H"], a["W"], x.cs, a["cin"], g.ptr(), a["Ho"], a["Wo"], g.cs,
                                     a["cout"], a["kh"], a["kw"], a["stride"], a["pad"], a["dil"], sc.data_ptr(), nb, dw,
                                     _stream())
    elif k == "bn_stats":
        C, n = a["C"], a["n"]
        rm, rv = (a["rm"].clone(), a["rv"].clone()) if a["rm"] is not None else (None, None)
        nb = L.stp3_bn_scratch_bytes(n, C)
        sc = _scratch(nb)
        ptrs = [out(nm, Out(1, C)) for nm in ("mean", "var", "invstd")]
        code = L.stp3_bn_stats(a["x"].ptr(), n, C, a["x"].cs, a["eps"], a["momentum"], rm.data_ptr() if rm is not None else None,
                               rv.data_ptr() if rv is not None else None, *ptrs, sc.data_ptr(), nb, _stream())
        if rm is not None:
            outs["run_mean"], outs["run_var"] = (None, rm, None), (None, rv, None)
    elif k == "bn_apply" and a["mode"] is not None:
        C, n, hl = a["C"], a["n"], a["hl_cs"]
        yp = out("y", a["y"])
        plane = torch.full((n * hl + 8,), SENT16, dtype=torch.int16, device=DEV).view(a["mode"])
        outs["plane"] = (None, plane, None)
        res = a["res"]
        code = L.stp3_bn_apply_plane(a["x"].ptr(), n, C, a["x"].cs, a["mean"].data_ptr(), a["invstd"].data_ptr(),
                                     a["gamma"].data_ptr(), a["beta"].data_ptr(), res.ptr() if res else None,
                                     res.cs if res else 0, int(a["relu"]), a["p"], a["seed"], a["offset"], yp, a["y"].cs,
                                     plane.data_ptr() + 2 * a["plane_shift"], hl, dense.PLANE_OPERAND[a["mode"]],
                                     _stream())
    elif k == "bn_apply":
        C, n, hl = a["C"], a["n"], a["hl_cs"]
        yp = out("y", a["y"]) if a["y"] is not None else None
        planes = None
        if hl:
            planes = [torch.full((n * hl + 8,), SENT, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
            outs["hi"], outs["lo"] = (None, planes[0], None), (None, planes[1], None)
        res = a["res"]
        code = L.stp3_bn_apply(a["x"].ptr(), n, C, a["x"].cs, a["mean"].data_ptr(), a["invstd"].data_ptr(),
                               a["gamma"].data_ptr(), a["beta"].data_ptr(), res.ptr() if res else None,
                               res.cs if res else 0, int(a["relu"]), a["p"], a["seed"], a["offset"], yp,
                               a["y"].cs if a["y"] is not None else 0, planes[0].data_ptr() if hl else None,
                               planes[1].data_ptr() if hl else None, hl, _stream())
    elif k == "bn_bwd_reduce":
        C, n = a["C"], a["n"]
        nb = L.stp3_bn_scratch_bytes(n, C)
        sc = _scratch(nb)
        y, x = a["y"], a["x"]
        sg = out("sum_g", Out(1, C))
        sgx = out("sum_gx", Out(1, C)) if x is not None else None
        code = L.stp3_bn_bwd_reduce(a["g"].ptr(), a["g"].cs, y.ptr() if y else None, y.cs if y else 0,
                                    x.ptr() if x else None, x.cs if x else 0,
                                    a["mean"].data_ptr() if x else None, a["invstd"].data_ptr() if x else None,
                                    n, C, sg, sgx, sc.data_ptr(), nb, _stream())
    elif k == "bn_bwd_apply":
        C, n, y = a["C"], a["n"], a["y"]
        dx = out("dx", a["dx"])
        gm = out("g_masked", a["gm"]) if a["gm"] is not None else None
        code = L.stp3_bn_bwd_apply(a["g"].ptr(), a["g"].cs, y.ptr() if y else None, y.cs if y else 0, a["x"].ptr(),
                                   a["x"].cs, a["mean"].data_ptr(), a["invstd"].data_ptr(), a["gamma"].data_ptr(),
                                   a["sum_g"].data_ptr(), a["sum_gx"].data_ptr(), n, C, dx, a["dx"].cs, gm,
                                   a["gm"].cs if a["gm"] is not None else 0, _stream())
    elif k == "ics":
        nb = L.stp3_image_channel_sums_scratch_bytes(a["n_img"], a["hw"], a["C"])
        sc = _scratch(nb)
        code = L.stp3_image_channel_sums(a["x"].ptr(), a["n_img"], a["hw"], a["C"], a["x"].cs,
                                         out("sums", Out(1, a["n_img"] * a["C"])), sc.data_ptr(), nb, _stream())
    elif k == "tpm":
        B, T, C = a["B"], a["T"], a["C"]
        o = out("out", Out(1, B * (T if a["adjoint"] else T + 1) * C))
        code = L.stp3_temporal_pair_mean(a["m"].data_ptr(), B, T, C, int(a["adjoint"]), o, _stream())
    elif k == "up":
        y = a["y"]
        out("y", y)                    # the API takes the base of the wide rows and the window offset apart
        base = outs["y"][1].data_ptr() + 4 * y.shift
        code = L.stp3_upsample2x_window_f32(a["x"].ptr(), a["n_img"], a["h"], a["w"], a["C"], base, y.cs, y.coff, _stream())
    elif k == "up_bwd":
        gy = a["gy"]
        o = out("gx", Out(1, a["n_img"] * a["h"] * a["w"] * a["C"], shift=a.get("gx_shift", 0)))
        code = L.stp3_upsample2x_window_bwd(gy.store.data_ptr() + 4 * gy.shift, gy.cs, gy.coff, a["n_img"], a["h"], a["w"], a["C"], o, _stream())
    elif k == "interleave":
        ph = [t.data_ptr() if t is not None else None for t in a["phases"]]
        o = out("out", Out(1, a["n_img"] * a["H"] * a["W"] * a["C"]))
        code = L.stp3_phase_interleave(*ph, a["n_img"], a["H"], a["W"], a["C"], o, _stream())
    elif k == "sigmoid":
        o = out("dz", Out(1, a["g"].numel()))
        code = L.stp3_sigmoid_bwd(a["g"].data_ptr(), a["s"].data_ptr(), a["g"].numel(), o, _stream())
    else:
        raise AssertionError(k)
    _lib.check(code, f"replay {k}")
    torch.cuda.synchronize()
    got = {nm: (spec.window(store) if spec is not None else store) for nm, (spec, store, keep) in outs.items()}
    return got, outs


# ------------------------------------------------------------------------------------------------ references and checks
def _ulps(got, ref, mag, k, rel=0.0):
    """max over elements of |got - ref| / (k ulps of mag + rel |ref|); <= 1 passes"""
    bar = k * ULP * mag + rel * ref.abs() + 1e-300
    return float(((got.double() - ref).abs() / bar).max())


def check(case: Case):
    """-> dict of measured quantities; raises nothing (the tests assert on the dict)"""
    a, k = case.a, case.kind
    got, outs = run(case)
    first = {nm: s.clone() for nm, (_, s, _) in outs.items()}
    got2, outs2 = run(case)
    res = {"same": all(torch.equal(first[nm].view(torch.uint8) if first[nm].dtype != torch.bool else first[nm],
                                   s.view(torch.uint8)) for nm, (_, s, _) in outs2.items()),
           "untouched": all(bool((s[keep] == SENT).all()) for _, s, keep in outs.values() if keep is not None)}
    if case.prod is not None:              # bitwise; the bf16 planes' storage ends in a guard the production one lacks
        bits = lambda t: t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)   # noqa: E731
        res["production"] = all(torch.equal(bits(got[nm])[:case.prod[nm].numel()], bits(case.prod[nm])) for nm in case.prod)
    ratios = {}
    if k == "wgrad":
        x = a["x"].vals.view(a["n_img"], a["H"], a["W"], a["cin"])
        g = a["g"].vals.view(a["n_img"], a["Ho"], a["Wo"], a["cout"])
        args = (a["kh"], a["kw"], a["stride"], a["pad"], a["dil"], a["kt"], a["T"])
        if a["mode"] is not None:       # one product of the plane values: the exact result is the model
            exact = model = R.wgrad(x, g, *args, plane=a["mode"])
        else:
            exact, model = R.wgrad(x, g, *args), R.wgrad(x, g, *args, model=True)
        dw = got["dw"].reshape(exact.shape).double()
        scale = max(float(exact.abs().max()), 1e-30)
        res["exact"] = float((dw - exact).abs().max()) / scale
        if a["n_img"] * a["Ho"] * a["Wo"] < 64 and a["mode"] is None:
            # a sum of fewer than 64 products (the squeeze-excite weights over one-pixel images) may cancel far below
            # its terms: there the bf16 x 3 representation (at most 2^-16 of each |x g|, the model above) is held to
            # the terms' summed magnitudes instead of the cancelled max
            mags = R.wgrad(x.abs(), g.abs(), *args)
            res["exact"] = min(res["exact"], float(((dw - exact).abs() / (2.0 ** -16 * mags + 1e-300)).max()) *
                               WGRAD_EXACT_BAR)
        res["model"] = float((dw - model).abs().max()) / scale
        res["per"] = a["per"]
        res["finite"] = bool(torch.isfinite(dw).all())
        dead = exact.abs().amax(dim=(0, 1)) == 0
        res["dead_exact_zero"] = not bool(dw.permute(2, 3, 4, 0, 1)[dead].any()) if case.features & {"dead tap"} else True
        ratios["exact"] = res["exact"] / WGRAD_EXACT_BAR
        ratios["model"] = res["model"] / wgrad_bar(a["per"])
    elif k == "bn_stats":
        ref = R.bn_stats(a["x"].vals, a["eps"], a["momentum"], a["rm"], a["rv"])
        ratios["mean"] = _ulps(got["mean"], ref["mean"], ref["abs_mean"], 2 ** -16, 2 * ULP)
        ratios["var"] = _ulps(got["var"], ref["var"], ref["sq_mean"], 2 ** -16, 2 * ULP)
        ratios["invstd"] = _ulps(got["invstd"], ref["invstd"], ref["invstd"], 4)
        if a["rm"] is not None:
            m = float(np.float32(a["momentum"]))
            mag_m = (1 - m) * a["rm"].double().abs() + m * ref["mean"].abs()
            mag_v = (1 - m) * a["rv"].double().abs() + m * ref["var"].abs() * 2
            ratios["run_mean"] = _ulps(got["run_mean"], ref["run_mean"], mag_m, 4)
            ratios["run_var"] = _ulps(got["run_var"], ref["run_var"], mag_v, 6)
    elif k == "bn_apply" and a["mode"] is not None:
        n, C, hl, sh = a["n"], a["C"], a["hl_cs"], a["plane_shift"]
        ref = R.bn_apply(a["x"].vals, a["mean"], a["invstd"], a["gamma"], a["beta"],
                         a["res"].vals if a["res"] else None, a["relu"], a["p"], a["seed"], a["offset"])
        y = got["y"]
        # y exactly as stp3_bn_apply stores it on the same arguments
        twin, _ = run(Case("bn_apply", dict(a, mode=None, hl_cs=0)))
        res["y_as_bn_apply"] = torch.equal(y.contiguous().view(torch.int32), twin["y"].contiguous().view(torch.int32))
        pl = got["plane"][sh:sh + n * hl].view(n, hl)
        want = R.bn_apply_plane(y.contiguous(), hl, a["mode"])
        res["plane_is_rounded_y"] = torch.equal(pl.view(torch.int16), want.view(torch.int16))
        res["padding +0"] = not bool(pl[:, C:].view(torch.int16).any())
        bits = got["plane"].view(torch.int16)
        res["guard"] = bool((bits[:sh] == SENT16).all() and (bits[sh + n * hl:] == SENT16).all())
        ratios["y"] = _ulps(y, ref["y"], ref["mag"], 8)
        if ref["keep"] is not None:
            res["dropped_zero"] = not bool(y[~ref["keep"]].any())
            res["keep_bits"] = not bool(((y == 0) & (ref["y"].abs() > 8 * ULP * ref["mag"])).any())
    elif k == "bn_apply":
        ref = R.bn_apply(a["x"].vals, a["mean"], a["invstd"], a["gamma"], a["beta"],
                         a["res"].vals if a["res"] else None, a["relu"], a["p"], a["seed"], a["offset"])
        n, C, hl = a["n"], a["C"], a["hl_cs"]
        y = got["y"] if a["y"] is not None else None
        if hl:
            hi = got["hi"][:n * hl].view(n, hl)
            lo = got["lo"][:n * hl].view(n, hl)
            res["padding_zero"] = bool((hi[:, C:] == 0).all() and (lo[:, C:] == 0).all()) and \
                not bool(torch.signbit(hi[:, C:].float()).any() or torch.signbit(lo[:, C:].float()).any())
            res["guard"] = bool((got["hi"][n * hl:] == torch.tensor(SENT, dtype=torch.bfloat16)).all())
            if y is not None:
                h2, l2 = dense.split_hilo(y.contiguous())
                res["planes_split_y"] = torch.equal(hi[:, :C].view(torch.int16), h2.view(torch.int16)) and \
                    torch.equal(lo[:, :C].view(torch.int16), l2.view(torch.int16))
            else:
                y = hi[:, :C].float() + lo[:, :C].float()
        ratios["y"] = _ulps(y, ref["y"], ref["mag"], 8, 2.0 ** -16 if a["y"] is None else 0.0)
        if ref["keep"] is not None:
            res["dropped_zero"] = not bool(y[~ref["keep"]].any())
            dropped_by_kernel = (y == 0) & (ref["y"].abs() > 8 * ULP * ref["mag"])
            res["keep_bits"] = not bool(dropped_by_kernel.any())
    elif k == "bn_bwd_reduce":
        ref = R.bn_bwd_reduce(a["g"].vals, a["y"].vals if a["y"] else None, a["x"].vals if a["x"] else None,
                              a["mean"], a["invstd"])
        ratios["sum_g"] = _ulps(got["sum_g"], ref["sum_g"], ref["mag_g"], 2 ** -16, 2 * ULP)
        if a["x"] is not None:
            ratios["sum_gx"] = _ulps(got["sum_gx"], ref["sum_gx"], ref["mag_gx"], 4, 2 * ULP)
    elif k == "bn_bwd_apply":
        yv = a["y"].vals if a["y"] else None
        ref = R.bn_bwd_apply(a["g"].vals, yv, a["x"].vals, a["mean"], a["invstd"], a["gamma"], a["sum_g"], a["sum_gx"])
        ratios["dx"] = _ulps(got["dx"], ref["dx"], ref["mag"], 8)
        if a["gm"] is not None:
            g = a["g"].vals
            want = torch.where(yv > 0, g, torch.zeros_like(g)) if yv is not None else g
            res["g_masked_bitwise"] = torch.equal(got["g_masked"].contiguous().view(torch.int32), want.view(torch.int32))
    elif k == "ics":
        ref = R.image_channel_sums(a["x"].vals.view(a["n_img"], a["hw"], a["C"]))
        ratios["sums"] = _ulps(got["sums"].view(a["n_img"], a["C"]), ref["sums"], ref["mag"], 2 ** -16, 2 * ULP)
    elif k == "tpm":
        B, T, C = a["B"], a["T"], a["C"]
        ref = R.temporal_pair_mean(a["m"].view(B, T + 1 if a["adjoint"] else T, C), a["adjoint"])
        ratios["out"] = _ulps(got["out"].view(ref["out"].shape), ref["out"], ref["mag"], 1)
    elif k == "up":
        ref = R.upsample2x(a["x"].vals.view(a["n_img"], a["h"], a["w"], a["C"]))
        ratios["y"] = _ulps(got["y"].reshape(ref["y"].shape), ref["y"], ref["mag"], 4)
    elif k == "up_bwd":
        ref = R.upsample2x_bwd(a["gy"].vals.view(a["n_img"], 2 * a["h"], 2 * a["w"], a["C"]))
        ratios["gx"] = _ulps(got["gx"].reshape(ref["gx"].shape), ref["gx"], ref["mag"], 6)
    elif k == "interleave":
        ref = R.phase_interleave(a["phases"], a["H"], a["W"])
        res["copy_bitwise"] = torch.equal(got["out"].reshape(ref.shape).view(torch.int32), ref.view(torch.int32))
    elif k == "sigmoid":
        ref = R.sigmoid_bwd(a["g"], a["s"])
        ratios["dz"] = _ulps(got["dz"].reshape(ref["dz"].shape), ref["dz"], ref["mag"], 4)
    res["ratios"] = ratios
    return res


def passed(res):
    flags = [v for kk, v in res.items() if isinstance(v, bool)]
    return all(flags) and all(r <= 1.0 for r in res["ratios"].values())


# ------------------------------------------------------------------------------------------------ case constructors
def wgrad_case(x, g, n_img, H, W, cin, Ho, Wo, cout, kh, kw, stride=1, pad=None, dil=1, kt=1, B=None, T=1,
               is3d=False, tag="", mode=None):
    """x, g: In (fp32), or PIn of the plane type `mode` (stp3_conv_wgrad_plane / stp3_conv3d_wgrad_plane)"""
    pad = (kh - 1) * dil // 2 if pad is None else pad
    a = dict(x=x, g=g, n_img=n_img, H=H, W=W, cin=cin, Ho=Ho, Wo=Wo, cout=cout, kh=kh, kw=kw, stride=stride, pad=pad,
             dil=dil, kt=kt, T=T, B=B if B is not None else n_img // T, is3d=is3d, mode=mode)
    P = n_img * Ho * Wo
    n, per = R.wgrad_split(P, kt * kh * kw, cout, cin)
    a["per"], a["n_split"] = per, n
    f = {"wgrad 3-D" if is3d else "wgrad 2-D"}
    if -(-P // per) < n:
        f.add("empty split")
    if stride == 2:
        f.add("stride 2")
    if dil > 1:
        f.add("dilation")
    if kt > 1:
        f.add("time taps")
        if a["B"] > 1:
            f.add("sample boundaries")
    if not (x.aligned() and g.aligned()):
        f.add("wgrad scalar loads")

    def live(d, n_out, n_in):
        o = 0 if d >= 0 else (-d + stride - 1) // stride
        return o < n_out and o * stride + d < n_in
    for it in range(kt):
        for ky in range(kh):
            for kx in range(kw):
                if not (live(ky * dil - pad, Ho, H) and live(kx * dil - pad, Wo, W) and kt - 1 - it < T):
                    f.add("dead tap")
    if mode is not None:
        f = {f"plane {v}" for v in f} | {f"plane wgrad {PLANE_NAMES[mode]}"}
        if P % 64 in (1, 63):
            f.add("plane P = 64k +- 1")
        if P < 64:
            f.add("plane P < 64")
    return Case("wgrad", a, tag, features=f)


PLANE_NAMES = {torch.float16: "fp16", torch.bfloat16: "bf16"}


def bn_apply_case(x: In, C, mean, invstd, gamma, beta, res=None, relu=False, p=0.0, seed=0, offset=0, y=None, hl_cs=0,
                  tag="", mode=None, plane_shift=0):
    """mode (torch.float16 / torch.bfloat16): stp3_bn_apply_plane, one plane of rows of hl_cs channels starting
    plane_shift elements into its storage"""
    n = x.vals.shape[0]
    a = dict(x=x, n=n, C=C, mean=mean, invstd=invstd, gamma=gamma, beta=beta, res=res, relu=relu, p=float(p), seed=seed,
             offset=offset, y=y, hl_cs=hl_cs, mode=mode, plane_shift=plane_shift)
    vec = C % 8 == 0 and x.aligned() and (res is None or res.aligned()) and (y is None or y.aligned())
    f = {"bn_apply vector" if vec else "bn_apply scalar"}
    if p > 0:
        f.add("dropout")
        if (offset + n * C) >> 32 != offset >> 32 or offset >> 32:
            f.add("dropout offset >= 2^32")
    if hl_cs > C:
        f.add("bf16 padding" if not vec else "bf16 padding, vector")
    if y is not None and y.cs > C:
        f.add("bn_apply window")
    if mode is not None:
        f = {f"plane {v}" for v in f if "bf16 padding" not in v} | {"bn_apply_plane", f"bn_apply_plane {PLANE_NAMES[mode]}"}
        if hl_cs > C:
            f.add("plane padding" + (", vector" if vec and hl_cs - C >= 8 else ""))
        if hl_cs % 64:
            f.add("plane plane_cstride not a multiple of 64")
    return Case("bn_apply", a, tag, features=f)


def bn_bwd_apply_case(g: In, y: Optional[In], x: In, C, mean, invstd, gamma, sum_g, sum_gx, dx: Out, gm: Optional[Out],
                      tag=""):
    n = x.vals.shape[0]
    a = dict(g=g, y=y, x=x, n=n, C=C, mean=mean, invstd=invstd, gamma=gamma, sum_g=sum_g, sum_gx=sum_gx, dx=dx, gm=gm)
    vec = C % 8 == 0 and g.aligned() and x.aligned() and dx.aligned() and (y is None or y.aligned()) and \
        (gm is None or gm.aligned())
    f = {"bn_bwd_apply vector" if vec else "bn_bwd_apply scalar"}
    if dx.cs > C:
        f.add("bn_bwd_apply window")
    if gm is not None:
        f.add("g_masked")
    return Case("bn_bwd_apply", a, tag, features=f)


def up_case(x: In, n_img, h, w, C, y: Out, tag=""):
    vec = C % 4 == 0 and y.cs % 4 == 0 and y.coff % 4 == 0 and x.aligned() and (y.shift + y.coff) % 4 == 0
    return Case("up", dict(x=x, n_img=n_img, h=h, w=w, C=C, y=y), tag,
                features={"upsample vector" if vec else "upsample scalar"} | ({"upsample window"} if y.cs > C else set()))


def up_bwd_case(gy: In, n_img, h, w, C, gx_shift=0, tag=""):
    vec = C % 4 == 0 and gy.cs % 4 == 0 and gy.coff % 4 == 0 and gy.aligned() and gx_shift % 4 == 0
    return Case("up_bwd", dict(gy=gy, n_img=n_img, h=h, w=w, C=C, gx_shift=gx_shift), tag,
                features={"upsample_bwd vector" if vec else "upsample_bwd scalar"} |
                ({"upsample_bwd window"} if gy.cs > C else set()))


# ------------------------------------------------------------------------------------------------ recording
class Recorder:
    """Wraps the dense_train entry points (every model caller looks them up as dense_train.<name>) and turns each call
    into Cases with cloned inputs and a clone of what production wrote."""
    NAMES = ("conv_wgrad", "bn_stats", "bn_apply", "bn_backward", "channel_sums", "image_channel_sums",
             "temporal_pair_mean", "upsample2x", "upsample2x_backward", "upsample2x_into", "upsample2x_backward_from",
             "phase_interleave", "sigmoid_backward")

    def __init__(self, source):
        self.source, self.cases = source, []

    def __enter__(self):
        self.mp = pytest.MonkeyPatch()
        for nm in self.NAMES:
            self.mp.setattr(dense_train, nm, self._wrap(nm, getattr(dense_train, nm)))
        return self

    def __exit__(self, *exc):
        self.mp.undo()
        torch.cuda.synchronize()

    def _add(self, case, prod):
        case.tag = f"{self.source}: {case.tag}"
        case.prod = {k: v.detach().clone() for k, v in prod.items()}
        case.features.add("plane recorded" if case.a.get("mode") is not None else "recorded")
        self.cases.append(case)

    def _wrap(self, nm, orig):
        rec = getattr(self, "_" + nm)

        def wrapper(*args, **kw):
            before = rec(*args, **kw)
            out = orig(*args, **kw)
            rec(*args, **kw, _after=(before, out))
            return out
        return wrapper

    # each _<name>(args, _after=None): called before the call (returns what must be cloned first) and after it
    def _conv_wgrad(self, x, g, kh, kw, stride, dilation=1, kt=None, mode=None, _after=None):
        if _after is None:
            return None
        dw = _after[1]
        if mode is not None:
            (xv, xcs, (H, W), bt_x), (gv, gcs, (Ho, Wo), bt_g) = _plane_operand(x, mode), _plane_operand(g, mode)
            cin, cout, N = xv.shape[-1], gv.shape[-1], xv.shape[0] // (H * W)
            name = PLANE_NAMES[mode]
            if kt is not None:
                B, T = bt_x or bt_g
                c = wgrad_case(PIn(xv, xcs), PIn(gv, gcs), N, H, W, cin, H, W, cout, kh, kw, 1, (kh - 1) // 2, 1, kt, B,
                               T, True, f"wgrad3d {name} ({kt},{kh},{kw}) {cin}->{cout} {B}x{T}x{H}x{W}", mode)
            else:
                c = wgrad_case(PIn(xv, xcs), PIn(gv, gcs), N, H, W, cin, Ho, Wo, cout, kh, kw, stride, None, dilation,
                               tag=f"wgrad {name} {kh}x{kw} s{stride} d{dilation} {cin}->{cout} {N}x{H}x{W}", mode=mode)
            self._add(c, {"dw": dw.reshape(-1)})
            return
        if x.dim() == 5:
            B, T, H, W, cin = x.shape
            cout = g.shape[-1]
            c = wgrad_case(In(x), In(g), B * T, H, W, cin, H, W, cout, kh, kw, 1, (kh - 1) // 2, 1, kt, B, T, True,
                           f"wgrad3d ({kt},{kh},{kw}) {cin}->{cout} {B}x{T}x{H}x{W}")
        else:
            N, H, W, cin = x.shape
            _, Ho, Wo, cout = g.shape
            c = wgrad_case(In(x), In(g), N, H, W, cin, Ho, Wo, cout, kh, kw, stride, None, dilation,
                           tag=f"wgrad {kh}x{kw} s{stride} d{dilation} {cin}->{cout} {N}x{H}x{W}")
            if H == W == 1 and N < 64:          # the trunk's squeeze-excite weights: one pixel per image
                c.features.add("wgrad P < 64, one-pixel images")
        self._add(c, {"dw": dw.reshape(-1)})

    def _bn_stats(self, x, eps, momentum, running_mean=None, running_var=None, _after=None):
        if _after is None:
            return (running_mean.clone() if running_mean is not None else None,
                    running_var.clone() if running_var is not None else None)
        (rm, rv), st = _after
        C = x.shape[-1]
        c = Case("bn_stats", dict(x=In_of(x), n=x.numel() // C, C=C, eps=float(eps), momentum=float(momentum), rm=rm, rv=rv),
                 f"bn_stats C{C} n{x.numel() // C}", features={"bn_stats"})
        prod = {"mean": st.mean, "var": st.var, "invstd": st.invstd}
        if rm is not None:
            prod.update(run_mean=running_mean, run_var=running_var)
        self._add(c, prod)

    def _bn_apply(self, x, st, gamma, beta, relu, res=None, hl=True, dropout=(0.0, 0, 0), y_out=None, mode=None,
                  _after=None):
        if _after is None:
            return None
        y, planes = _after[1]
        N, H, W, C = x.shape
        cs = dense_train._row_stride(y)
        ys = Out(N * H * W, C, cs, y.storage_offset() % cs)
        p, seed, offset = dropout
        c = bn_apply_case(In_of(x), C, _vec(st.mean), _vec(st.invstd), _vec(gamma), _vec(beta),
                          In_of(res) if res is not None else None, relu, p, int(seed), int(offset), ys,
                          planes.hi.shape[-1] if planes is not None else 0, f"bn_apply C{C} n{N * H * W} p{p}",
                          mode if planes is not None else None)
        prod = {"y": y.reshape(-1, C)}
        if planes is not None and mode is not None:
            prod["plane"] = planes.hi.reshape(-1)
        elif planes is not None:
            prod.update(hi=planes.hi.reshape(-1), lo=planes.lo.reshape(-1))
        self._add(c, prod)

    def _bn_backward(self, g, x, st, gamma, y_mask, want_masked=False, dx_out=None, _after=None):
        if _after is None:
            return None
        dx, sum_gx, sum_g, gm = _after[1]
        N, H, W, C = x.shape
        n = N * H * W
        yi = In_of(y_mask) if y_mask is not None else None
        red = Case("bn_bwd_reduce", dict(g=In_of(g), y=yi, x=In_of(x), mean=_vec(st.mean), invstd=_vec(st.invstd), n=n, C=C),
                   f"bn_bwd_reduce C{C} n{n}", features={"bn_bwd_reduce", "relu mask"} if y_mask is not None else {"bn_bwd_reduce"})
        if y_mask is None and n > 10 ** 5:
            red.features.add("unmasked bn_backward, n > 1e5")
        self._add(red, {"sum_g": sum_g, "sum_gx": sum_gx})
        cs = dense_train._row_stride(dx)
        c = bn_bwd_apply_case(In_of(g), yi, In_of(x), C, _vec(st.mean), _vec(st.invstd), _vec(gamma), _vec(sum_g),
                              _vec(sum_gx), Out(n, C, cs, dx.storage_offset() % cs), Out(n, C) if want_masked else None,
                              f"bn_bwd_apply C{C} n{n}")
        if y_mask is None and n > 10 ** 5:
            c.features.add("unmasked bn_backward, n > 1e5")
        prod = {"dx": dx.reshape(-1, C)}
        if want_masked:
            prod["g_masked"] = gm.reshape(-1, C)
        self._add(c, prod)

    def _channel_sums(self, g, _after=None):
        if _after is None:
            return None
        C = g.shape[-1]
        c = Case("bn_bwd_reduce", dict(g=In_of(g), y=None, x=None, mean=None, invstd=None, n=g.numel() // C, C=C),
                 f"channel_sums {tuple(g.shape)}", features={"bn_bwd_reduce", "channel_sums"})
        if g.dim() == 4 and g.shape[1] == g.shape[2] == 1:
            c.features.add("channel_sums (M, 1, 1, C)")
        self._add(c, {"sum_g": _after[1]})

    def _image_channel_sums(self, x, _after=None):
        if _after is None:
            return None
        N, H, W, C = x.shape
        self._add(Case("ics", dict(x=In_of(x), n_img=N, hw=H * W, C=C), f"image_channel_sums {N}x{H * W}x{C}",
                       features={"image_channel_sums"}), {"sums": _after[1].reshape(-1)})

    def _temporal_pair_mean(self, m, T, adjoint=False, _after=None):
        if _after is None:
            return None
        B = m.shape[0] // (T + 1 if adjoint else T)
        self._add(Case("tpm", dict(m=_vec(m), B=B, T=T, C=m.shape[1], adjoint=bool(adjoint)), f"pair_mean adj{int(adjoint)}",
                       features={f"temporal_pair_mean adjoint {int(bool(adjoint))}"}), {"out": _after[1].reshape(-1)})

    def _upsample2x(self, x, _after=None):
        if _after is None:
            return None
        N, h, w, C = x.shape
        self._add(up_case(In(x), N, h, w, C, Out(N * 4 * h * w, C), f"upsample {N}x{h}x{w}x{C}"),
                  {"y": _after[1].reshape(-1, C)})

    def _upsample2x_into(self, x, y, coff, _after=None):
        if _after is None:
            return None
        N, h, w, C = x.shape
        Cy = y.shape[3]
        self._add(up_case(In(x), N, h, w, C, Out(N * 4 * h * w, C, Cy, coff), f"upsample_into {C}@{coff}/{Cy}"),
                  {"y": y.reshape(-1, Cy)[:, coff:coff + C]})

    def _upsample2x_backward(self, gy, _after=None):
        if _after is None:
            return None
        N, H2, W2, C = gy.shape
        self._add(up_bwd_case(In(gy), N, H2 // 2, W2 // 2, C, tag=f"upsample_bwd {N}x{H2}x{W2}x{C}"),
                  {"gx": _after[1].reshape(-1)})

    def _upsample2x_backward_from(self, gy, coff, C, _after=None):
        if _after is None:
            return None
        N, H2, W2, Cy = gy.shape
        gi = In(gy.reshape(-1, Cy)[:, coff:coff + C], Cy, coff)
        self._add(up_bwd_case(gi, N, H2 // 2, W2 // 2, C, tag=f"upsample_bwd_from {C}@{coff}/{Cy}"),
                  {"gx": _after[1].reshape(-1)})

    def _phase_interleave(self, phases, H, W, _after=None):
        if _after is None:
            return None
        ref = next(t for t in phases if t is not None)
        self._add(Case("interleave", dict(phases=[_vec(t) if t is not None else None for t in phases], n_img=ref.shape[0],
                                          H=H, W=W, C=ref.shape[-1]), f"interleave {H}x{W}",
                       features={"phase_interleave"} | ({"NULL phase"} if any(t is None for t in phases) else set())),
                  {"out": _after[1].reshape(-1)})

    def _sigmoid_backward(self, g, s, _after=None):
        if _after is None:
            return None
        self._add(Case("sigmoid", dict(g=_vec(g).reshape(-1), s=_vec(s).reshape(-1)), "sigmoid_bwd",
                       features={"sigmoid_bwd"}), {"dz": _after[1].reshape(-1)})


def train_entry_points_called_outside_dense_train():
    """Calls of a train-mode entry point of the library (the functions wrapped by dense_train) from any module of the
    package other than dense_train.py: they would bypass the Recorder."""
    names = {"stp3_conv_wgrad", "stp3_conv3d_wgrad", "stp3_bn_stats", "stp3_bn_apply", "stp3_bn_bwd_reduce",
             "stp3_bn_bwd_apply", "stp3_image_channel_sums", "stp3_temporal_pair_mean", "stp3_upsample2x_f32",
             "stp3_upsample2x_bwd", "stp3_upsample2x_window_f32", "stp3_upsample2x_window_bwd", "stp3_phase_interleave",
             "stp3_sigmoid_bwd", "stp3_conv_wgrad_plane", "stp3_conv3d_wgrad_plane", "stp3_bn_apply_plane"}
    pkg = os.path.dirname(os.path.abspath(dense_train.__file__))
    bad = []
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py") and os.path.join(root, f) != os.path.abspath(dense_train.__file__):
                with open(os.path.join(root, f)) as fh:
                    tree = ast.parse(fh.read())
                bad += [f"{f}:{n.lineno}" for n in ast.walk(tree) if isinstance(n, ast.Attribute) and n.attr in names]
    # inside dense_train.py every entry point is called from the function the Recorder wraps, or from
    # _conv_wgrad_plane provided the wrapped conv_wgrad is its only caller
    tree = ast.parse(inspect.getsource(dense_train))
    wrapped = set(Recorder.NAMES)
    helper = "_conv_wgrad_plane"
    callers = {fn.name for fn in tree.body if isinstance(fn, ast.FunctionDef)
               for n in ast.walk(fn) if isinstance(n, ast.Name) and n.id == helper}
    if callers != {"conv_wgrad"}:
        bad.append(f"dense_train.{helper} referenced from {sorted(callers)}, not only from conv_wgrad")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py") and os.path.join(root, f) != os.path.abspath(dense_train.__file__):
                with open(os.path.join(root, f)) as fh:
                    bad += [f"{f}:{n.lineno}" for n in ast.walk(ast.parse(fh.read()))
                            if isinstance(n, (ast.Attribute, ast.Name)) and getattr(n, "attr", getattr(n, "id", "")) == helper]
    for fn in tree.body:
        if isinstance(fn, ast.FunctionDef) and fn.name not in wrapped | {helper}:
            bad += [f"dense_train.{fn.name}:{n.lineno}" for n in ast.walk(fn) if isinstance(n, ast.Attribute) and n.attr in names]
    return bad


# ------------------------------------------------------------------------------------------------ the models' launches
def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def _step(fwd, seed, mode=None):
    """run fwd() -> outputs, then backward of sum(out * G) with G from `seed`.  mode (torch.float16 / torch.bfloat16):
    the forward under torch.autocast of that type and the backward outside it, as a precision-16 trainer runs a step"""
    with torch.autocast("cuda", dtype=mode or torch.float16, enabled=mode is not None):
        out = fwd()
    outs = [v for v in (out.values() if isinstance(out, dict) else [out]) if v is not None]
    gen = torch.Generator().manual_seed(seed)
    sum((v.float() * torch.randn(v.shape, generator=gen).to(DEV)).sum() for v in outs).backward()


# One train step of each module; the rec_* functions record it with this file's Recorder, and the convolution and
# helper suites run the same steps (under autocast too) inside their own recorders.
def decoder_step(shape, gates, mode=None):
    from stp3_b200.models.decoder import Decoder
    dec = TD.init_exact(Decoder(64, 2, 3, 2, gates), seed=2).train().to(DEV)
    x = gauss(shape, 6).to(DEV).requires_grad_(True)
    _step(lambda: dec(x), 9, mode)


def deeplab_step(cin, ncls, hidden, N, H, W, mode=None):
    from stp3_b200.layers.convolutions import DeepLabHead
    head = TD.init_exact(DeepLabHead(cin, ncls, hidden_channel=hidden), seed=3).train().to(DEV)
    x = gauss((N, cin, H, W), 4).to(DEV).requires_grad_(True)
    torch.manual_seed(5)
    _step(lambda: head(x), 6, mode)


def temporal_step(cin, nc, S, B, H, W, mode=None):
    from stp3_b200.models.temporal_model import TemporalModel
    tm = TD.init_exact(TemporalModel(cin, S, (H, W), start_out_channels=64), seed=3)
    tm.model[0].n_const = nc
    tm = tm.train().to(DEV)
    x = gauss((B, S, cin - nc, H, W), 5).to(DEV).requires_grad_(True)
    const = gauss((B * S, nc), 6).to(DEV) if nc else None
    torch.manual_seed(7)
    _step(lambda: tm(x, const=const), 8, mode)


def encoder_heads_step(name, mode=None):
    from oracle import make_golden_encoder_train as MG
    from stp3_b200.layers import convolutions as CV
    head, up, mods = MG.make_modules(CV, name)
    mods.to(DEV)
    r_lo, r_hi = (t.to(DEV).requires_grad_(True) for t in MG.endpoints())
    torch.manual_seed(17)
    _step(lambda: up(head(r_hi) if head is not None else r_hi, r_lo), 18, mode)


def trunk_step(version, M, H, W):
    """One train step of the opt-in trainable EfficientNet trunk (EfficientNetTrunk(version, trainable=True)) on M seeded
    H x W images: the oracle's seeded weights, the drop-connect draws after torch.manual_seed(5), the backward of
    sum(r3^2) + sum(r4).  The trunk ignores autocast, so it has no one-plane variant."""
    from oracle import efficientnet_oracle as EO
    from stp3_b200.models import efficientnet as EN
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=3), version)
    nat = EN.EfficientNetTrunk(version, trainable=True)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to(DEV).train()
    x = torch.randn(M, 3, H, W, generator=torch.Generator().manual_seed(1)).to(DEV)
    torch.manual_seed(5)
    r3, r4 = nat(x)
    (r3.square().sum() + r4.sum()).backward()
    torch.cuda.synchronize()


# The trunk steps every launch-by-launch suite replays: b0 and b4 on a small image (stem output 17 x 25), and b4 on one
# frame of six 224 x 480 cameras, where the partitioned reductions reach their part cap and ragged last parts.
TRUNK_STEPS = {"trunk_b0_35x51": ("b0", 3, 35, 51), "trunk_b4_35x51": ("b4", 3, 35, 51),
               "trunk_b4_224x480": ("b4", 6, 224, 480)}


def rec_decoder(shape, gates, name):
    with Recorder(name) as r:
        decoder_step(shape, gates)
    return r.cases


def rec_deeplab(cin, ncls, hidden, N, H, W, name):
    with Recorder(name) as r:
        deeplab_step(cin, ncls, hidden, N, H, W)
    return r.cases


def rec_temporal(cin, nc, S, B, H, W, name):
    with Recorder(name) as r:
        temporal_step(cin, nc, S, B, H, W)
    return r.cases


def rec_encoder_heads(name):
    with Recorder(f"encoder heads {name}") as r:
        encoder_heads_step(name)
    return r.cases


def rec_trunk(name):
    with Recorder(name) as r:
        trunk_step(*TRUNK_STEPS[name])
    return r.cases


GATES_ALL = dict(perceive_hdmap=True, predict_pedestrian=True, predict_instance=True, predict_future_flow=True,
                 planning=True)


# ------------------------------------------------------------------------------------------------ synthetic launches
def _r(*shape, seed, scale=1.0):
    return gauss(shape, seed) * scale


def synth_wgrad():
    cases = []

    def add(n_img, H, W, cin, cout, k, stride=1, dil=1, x_cs=0, g_cs=0, x_shift=0, g_shift=0, tag="", kt=1, T=1):
        Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
        x = In(_r(n_img * H * W, cin, seed=len(cases) * 2 + 1), x_cs, 0, x_shift)
        g = In(_r(n_img * Ho * Wo, cout, seed=len(cases) * 2 + 2), g_cs, 0, g_shift)
        if kt > 1 or T > 1:
            cases.append(wgrad_case(x, g, n_img, H, W, cin, H, W, cout, k, k, 1, (k - 1) // 2, 1, kt, n_img // T, T, True, tag))
        else:
            cases.append(wgrad_case(x, g, n_img, H, W, cin, Ho, Wo, cout, k, k, stride, None, dil, tag=tag))
    add(2, 9, 11, 70, 40, 3, x_cs=72, g_cs=48, tag="wide rows")
    add(1, 13, 7, 33, 65, 3, x_cs=37, g_cs=67, tag="odd row strides (scalar loads)")
    add(1, 12, 10, 64, 64, 3, x_shift=1, g_shift=3, tag="pointers off by 4 / 12 bytes")
    for c in (1, 8, 63, 65, 129, 200):
        add(1, 10, 12, c, 200 if c == 1 else c + 1 if c < 200 else 8, 3, tag=f"cin {c}")
    add(1, 7, 9, 64, 64, 1, tag="P < 64")
    add(1, 43, 3, 16, 16, 1, tag="P = 64k + 1")
    add(1, 3, 85, 16, 16, 1, tag="P = 64k - 1")
    add(1, 127, 65, 16, 16, 1, tag="P = 64k - 1, several stages")
    add(2, 1, 77, 24, 40, 3, tag="1 x W")
    add(2, 61, 1, 24, 40, 3, tag="H x 1")
    add(2, 37, 29, 64, 48, 7, 2, tag="7x7 stride 2 odd")
    add(1, 40, 30, 32, 64, 7, 2, tag="7x7 stride 2 even")
    add(1, 21, 15, 64, 64, 3, 2, tag="3x3 stride 2 odd")
    add(1, 19, 43, 64, 64, 3, 1, 12, tag="dilation 12, taps partly in padding")
    add(2, 9, 30, 64, 64, 3, 1, 12, tag="dilation 12, row taps wholly in padding")
    add(1, 11, 7, 40, 40, 3, 1, 36, tag="dilation 36 > H, W: only the centre tap lives")
    add(2, 130, 130, 128, 128, 1, tag="empty trailing splits")
    add(1, 9, 10, 35, 35, 3, kt=2, T=1, tag="3-D T = 1, kt = 2 (dead time tap)")
    add(2, 6, 5, 35, 35, 3, kt=3, T=2, tag="3-D T < kt, B = 2")
    add(3, 11, 13, 40, 24, 3, kt=2, T=3, tag="3-D B = 1, T = 3")
    add(6, 14, 12, 64, 64, 1, kt=2, T=3, tag="3-D (2,1,1), B = 2")
    add(4, 16, 16, 64, 64, 3, kt=2, T=2, x_cs=68, g_cs=65, tag="3-D wide / odd rows, B = 2")
    return cases


def synth_bn():
    cases = []
    for C, n, xcs, coff, shift, p, seed, off, relu, res, hl in [
            (1, 300, 1, 0, 0, 0.0, 0, 0, True, False, 8),
            (7, 1000, 9, 1, 0, 0.3, (5 << 32) | 11, 2 ** 32 - 3000, True, True, 8),
            (33, 127, 40, 3, 1, 0.0, 0, 0, False, True, 64),
            (1030, 129, 1030, 0, 0, 0.5, 77, 2 ** 33 + 5, True, False, 1088),
            (64, 100, 64, 0, 0, 0.1, (1 << 40) + 3, 2 ** 32 - 64 * 50, True, True, 64),
            (64, 5000, 72, 8, 0, 0.0, 0, 0, True, True, 128),
            (128, 256, 256, 128, 0, 0.5, 9, 12345, True, False, 192),
            (16, 1, 16, 0, 0, 0.0, 0, 0, False, False, 16)]:
        k = len(cases)
        x = In(_r(n, C, seed=100 + k, scale=3.0) + 0.5, xcs, coff, shift)
        mean = _r(C, seed=200 + k).to(DEV)
        invstd = (_r(C, seed=300 + k).abs() + 0.2).to(DEV)
        gamma, beta = _r(C, seed=400 + k).to(DEV), _r(C, seed=500 + k, scale=0.3).to(DEV)
        r = In(_r(n, C, seed=600 + k), xcs + 1, 1) if res else None
        y = Out(n, C, xcs + 3, 2, shift) if k % 2 else Out(n, C)
        cases.append(bn_apply_case(x, C, mean, invstd, gamma, beta, r, relu, p, seed, off, y, hl,
                                   f"bn_apply C{C} n{n} cs{xcs}@{coff}+{shift} p{p} off{off:#x}"))
        # statistics of the same rows, with running buffers
        rm, rv = _r(C, seed=700 + k).to(DEV), (_r(C, seed=800 + k).abs() + 0.5).to(DEV)
        cases.append(Case("bn_stats", dict(x=x, n=n, C=C, eps=1e-5, momentum=0.1, rm=rm if k % 3 else None,
                                           rv=rv if k % 3 else None), f"bn_stats C{C} n{n}", features={"bn_stats"}))
        # backward
        g = In(_r(n, C, seed=900 + k), xcs, coff, shift)
        ymask = In(_r(n, C, seed=1000 + k), xcs + 1, 0) if relu else None
        cases.append(Case("bn_bwd_reduce", dict(g=g, y=ymask, x=x, mean=mean, invstd=invstd, n=n, C=C),
                          f"bn_bwd_reduce C{C} n{n}", features={"bn_bwd_reduce"} | ({"relu mask"} if relu else set())))
        sg, sgx = _r(C, seed=1100 + k, scale=30.0).to(DEV), _r(C, seed=1200 + k, scale=30.0).to(DEV)
        cases.append(bn_bwd_apply_case(g, ymask, x, C, mean, invstd, gamma, sg, sgx,
                                       Out(n, C, 4 * C + 1, C + 1, shift) if k % 2 else Out(n, C, 4 * C, C),
                                       Out(n, C, C + 2, 1) if relu else None, f"bn_bwd_apply C{C} n{n}"))
        cases.append(Case("ics", dict(x=x, n_img=1 if n < 4 else 4 if n % 4 == 0 else 1,
                                      hw=n if n < 4 or n % 4 else n // 4, C=C), f"ics C{C}", features={"image_channel_sums"}))
    return cases


def synth_wgrad_plane():
    """plane weight gradients (both types) the modules never launch: odd row strides and pointers off 16 bytes (the
    scalar loads), channel counts 1 to 200, P < 64 and P = 64k +- 1, one-row / one-column maps, 7x7 and 3x3 stride 2 on
    odd and even maps, dilations with dead taps, empty trailing splits, 3-D with T = 1, T < kt and (2, 1, 1)"""
    cases = []
    for mode in PLANE_NAMES:
        def add(n_img, H, W, cin, cout, k, stride=1, dil=1, x_cs=0, g_cs=0, x_shift=0, g_shift=0, tag="", kt=1, T=1):
            s = len(cases)
            Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
            x = PIn(_r(n_img * H * W, cin, seed=3000 + 2 * s).to(mode), x_cs or dense.pad_to(cin), x_shift)
            g = PIn(_r(n_img * Ho * Wo, cout, seed=3001 + 2 * s).to(mode), g_cs or dense.pad_to(cout), g_shift)
            tag = f"{PLANE_NAMES[mode]} {tag}"
            if kt > 1 or T > 1:
                cases.append(wgrad_case(x, g, n_img, H, W, cin, H, W, cout, k, k, 1, (k - 1) // 2, 1, kt, n_img // T, T,
                                        True, tag, mode))
            else:
                cases.append(wgrad_case(x, g, n_img, H, W, cin, Ho, Wo, cout, k, k, stride, None, dil, tag=tag, mode=mode))
        add(2, 9, 11, 35, 40, 3, x_cs=37, g_cs=41, tag="row strides 37 / 41 (scalar loads)")
        add(1, 8, 9, 64, 64, 3, x_shift=1, g_shift=3, tag="pointers off by 2 / 6 bytes (scalar loads)")
        for cin in (1, 8, 63, 65, 129, 200):
            add(1, 10, 12, cin, 24, 3, tag=f"cin {cin}")
        add(1, 5, 7, 16, 16, 3, tag="P = 35 < 64")
        add(1, 5, 13, 16, 16, 3, tag="P = 65 = 64 + 1")
        add(1, 127, 65, 16, 16, 1, tag="P = 64k - 1, several stages")
        add(2, 1, 77, 24, 40, 3, tag="1 x W")
        add(2, 61, 1, 24, 40, 3, tag="H x 1")
        add(2, 37, 29, 64, 48, 7, 2, tag="7x7 stride 2 odd")
        add(1, 40, 30, 32, 64, 7, 2, tag="7x7 stride 2 even")
        add(1, 21, 15, 64, 64, 3, 2, tag="3x3 stride 2 odd")
        add(1, 20, 14, 64, 64, 3, 2, tag="3x3 stride 2 even")
        add(1, 19, 43, 64, 64, 3, 1, 12, tag="dilation 12, taps partly in padding")
        add(1, 11, 7, 40, 40, 3, 1, 36, tag="dilation 36 > H, W: only the centre tap lives")
        add(2, 130, 130, 128, 128, 1, tag="empty trailing splits")
        add(1, 9, 10, 35, 35, 3, kt=2, T=1, tag="3-D T = 1, kt = 2 (dead time tap)")
        add(2, 6, 5, 35, 35, 3, kt=3, T=2, tag="3-D T < kt")
        add(6, 14, 12, 64, 64, 1, kt=2, T=3, tag="3-D (2,1,1), B = 2")
    return cases


def synth_bn_plane():
    """stp3_bn_apply_plane (both types): C = 1, 7, 33, 64, 1030, input and output windows, residuals, dropout offsets
    at and past 2^32, plane row strides that are not multiples of 64, a plane starting 16 bytes into its storage"""
    cases = []
    for mode in PLANE_NAMES:
        for C, n, xcs, coff, shift, p, seed, off, relu, res, hl, psh in [
                (1, 300, 1, 0, 0, 0.0, 0, 0, True, False, 8, 0),
                (7, 1000, 9, 1, 0, 0.3, (5 << 32) | 11, 2 ** 32 - 3000, True, True, 16, 8),
                (33, 127, 40, 3, 1, 0.0, 0, 0, False, True, 40, 0),
                (1030, 129, 1030, 0, 0, 0.5, 77, 2 ** 33 + 5, True, False, 1088, 0),
                (64, 100, 64, 0, 0, 0.1, (1 << 40) + 3, 2 ** 32 - 64 * 50, True, True, 72, 8),
                (64, 5000, 72, 8, 0, 0.0, 0, 0, True, True, 128, 0),
                (40, 300, 40, 0, 0, 0.2, 5, 2 ** 32 + 7, True, False, 64, 0),
                (64, 200, 64, 0, 0, 0.0, 0, 0, False, False, 128, 8)]:
            k = len(cases)
            x = In(_r(n, C, seed=4000 + k, scale=3.0) + 0.5, xcs, coff, shift)
            mean = _r(C, seed=4100 + k).to(DEV)
            invstd = (_r(C, seed=4200 + k).abs() + 0.2).to(DEV)
            gamma, beta = _r(C, seed=4300 + k).to(DEV), _r(C, seed=4400 + k, scale=0.3).to(DEV)
            r = In(_r(n, C, seed=4500 + k), xcs + 1, 1) if res else None
            y = Out(n, C, xcs + 3, 2, shift) if k % 2 and k % 8 < 6 else Out(n, C)
            cases.append(bn_apply_case(x, C, mean, invstd, gamma, beta, r, relu, p, seed, off, y, hl,
                                       f"bn_apply_plane {PLANE_NAMES[mode]} C{C} n{n} cs{xcs}@{coff}+{shift} p{p} "
                                       f"off{off:#x} plane cs{hl}+{psh}", mode, psh))
    return cases


def synth_small():
    cases = []
    for n_img, h, w, C, cs, coff, shift in [(2, 5, 7, 12, 40, 4, 0), (1, 1, 9, 8, 8, 0, 0), (3, 6, 1, 5, 9, 3, 0),
                                            (1, 1, 1, 4, 12, 8, 1), (2, 4, 4, 64, 120, 56, 0)]:
        k = len(cases)
        cases.append(up_case(In(_r(n_img * h * w, C, seed=1300 + k)), n_img, h, w, C,
                             Out(n_img * 4 * h * w, C, cs, coff, shift), f"upsample {h}x{w} C{C} @{coff}/{cs}+{shift}"))
        gy = In(_r(n_img * 4 * h * w, C, seed=1400 + k), cs, coff, shift)
        cases.append(up_bwd_case(gy, n_img, h, w, C, 1 if k == 3 else 0, f"upsample_bwd {h}x{w} C{C} @{coff}/{cs}"))
    for H, W, null in [(9, 7, None), (10, 6, 1), (5, 1, 3), (1, 1, None)]:
        full = _r(2, H, W, 11, seed=1500 + H).to(DEV)
        ph = [full[:, py::2, px::2].contiguous() for py in range(2) for px in range(2)]
        ph = [None if (i == null or t.numel() == 0) else t for i, t in enumerate(ph)]
        cases.append(Case("interleave", dict(phases=ph, n_img=2, H=H, W=W, C=11), f"interleave {H}x{W} null {null}",
                          features={"phase_interleave"} | ({"NULL phase"} if None in ph else set())))
    for B, T, C, adj in [(2, 1, 5, 0), (2, 1, 5, 1), (3, 4, 33, 0), (3, 4, 33, 1)]:
        cases.append(Case("tpm", dict(m=_r(B * (T + adj), C, seed=1600 + T).to(DEV), B=B, T=T, C=C, adjoint=bool(adj)),
                          f"pair_mean B{B} T{T} adj{adj}", features={f"temporal_pair_mean adjoint {adj}"}))
    s = torch.sigmoid(_r(1001, seed=1700, scale=8.0)).to(DEV)
    cases.append(Case("sigmoid", dict(g=_r(1001, seed=1701).to(DEV), s=s), "sigmoid_bwd 1001", features={"sigmoid_bwd"}))
    return cases


SOURCES = {
    "decoder_48x64": lambda: rec_decoder((2, 3, 64, 48, 64), GATES_ALL, "decoder all gates 48x64"),
    "decoder_200x200": lambda: rec_decoder((2, 3, 64, 200, 200), dict(GATES_ALL, predict_instance=False,
                                                                     predict_future_flow=False, planning=False),
                                           "decoder B2 S3 200x200"),
    "deeplab_temporal_48x64": lambda: rec_deeplab(64, 64, 128, 6, 48, 64, "deeplab temporal_48x64"),
    "deeplab_encoder_14x30": lambda: rec_deeplab(160, 160, 64, 18, 14, 30, "deeplab encoder_14x30"),
    "temporal_perceive_ego_48x64": lambda: rec_temporal(70, 6, 3, 2, 48, 64, "temporal perceive_ego_48x64"),
    "temporal_perceive_ego_200x200": lambda: rec_temporal(70, 6, 3, 2, 200, 200, "temporal perceive_ego_200x200"),
    "temporal_stress_16x24": lambda: rec_temporal(134, 0, 5, 1, 16, 24, "temporal stress_16x24"),
    "encoder_heads_feat": lambda: rec_encoder_heads("feat"),
    "encoder_heads_uc": lambda: rec_encoder_heads("uc"),
    "synthetic_wgrad": synth_wgrad,
    "synthetic_bn": synth_bn,
    "synthetic_small": synth_small,
    "synthetic_wgrad_plane": synth_wgrad_plane,
    "synthetic_bn_plane": synth_bn_plane,
}


def rec_amp(mode, step, *args):
    """a step of one module with its forward under torch.autocast(dtype=mode)"""
    with Recorder(f"{step} {args[-1] if isinstance(args[-1], str) else args} {PLANE_NAMES[mode]}") as r:
        globals()[step](*args, mode=mode)
    return r.cases


for _m, _nm in PLANE_NAMES.items():
    SOURCES.update({
        f"amp_decoder_48x64_{_nm}": lambda m=_m: rec_amp(m, "decoder_step", (2, 3, 64, 48, 64), GATES_ALL),
        f"amp_deeplab_temporal_48x64_{_nm}": lambda m=_m: rec_amp(m, "deeplab_step", 64, 64, 128, 6, 48, 64),
        f"amp_deeplab_encoder_14x30_{_nm}": lambda m=_m: rec_amp(m, "deeplab_step", 160, 160, 64, 18, 14, 30),
        f"amp_temporal_48x64_{_nm}": lambda m=_m: rec_amp(m, "temporal_step", 70, 6, 3, 2, 48, 64),
        f"amp_encoder_heads_feat_{_nm}": lambda m=_m: rec_amp(m, "encoder_heads_step", "feat"),
        f"amp_encoder_heads_uc_{_nm}": lambda m=_m: rec_amp(m, "encoder_heads_step", "uc")})
SOURCES["amp_temporal_200x200_fp16"] = lambda: rec_amp(torch.float16, "temporal_step", 70, 6, 3, 2, 200, 200)
SOURCES.update({_nm: (lambda n=_nm: rec_trunk(n)) for _nm in TRUNK_STEPS})

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
        del r
    del cases
    torch.cuda.empty_cache()
    print(f"\n{name}: {len(rows)} launches in {time.time() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated")
    _RUNS[name] = rows
    return rows


def _fmt(r):
    res = r["res"]
    s = " ".join(f"{k} {v:.2f}" for k, v in res["ratios"].items())
    if r["kind"] == "wgrad":
        s = f"per {res['per']:5d}  exact {res['exact']:.2e}  model {res['model']:.2e}  ({s})"
    flags = [k for k, v in res.items() if isinstance(v, bool) and not v]
    return f"  {r['kind']:<13s} {r['tag'][:70]:<70s} {s}" + (f"  FAILED {flags}" if flags else "")


def test_no_train_entry_point_bypasses_the_recorder():
    assert not train_entry_points_called_outside_dense_train()


@pytest.mark.parametrize("name", list(SOURCES))
def test_train_launches_against_the_fp64_contract(name):
    rows = run_source(name)
    for r in rows:
        print(_fmt(r))
    bad = [_fmt(r) for r in rows if not r["ok"]]
    assert not bad, "\n".join(bad)


REQUIRED = ["recorded", "wgrad 2-D", "wgrad 3-D", "wgrad scalar loads", "dead tap", "empty split", "stride 2", "dilation",
            "time taps", "sample boundaries", "bn_stats", "bn_apply vector", "bn_apply scalar", "dropout",
            "dropout offset >= 2^32", "bf16 padding", "bf16 padding, vector", "bn_apply window", "bn_bwd_reduce", "relu mask", "channel_sums",
            "bn_bwd_apply vector", "bn_bwd_apply scalar", "bn_bwd_apply window", "g_masked", "image_channel_sums",
            "temporal_pair_mean adjoint 0", "temporal_pair_mean adjoint 1", "upsample vector", "upsample scalar",
            "upsample window", "upsample_bwd vector", "upsample_bwd scalar", "upsample_bwd window", "phase_interleave",
            "NULL phase", "sigmoid_bwd"]
REQUIRED += ["wgrad P < 64, one-pixel images", "unmasked bn_backward, n > 1e5", "channel_sums (M, 1, 1, C)"]
REQUIRED += ["plane recorded", "plane wgrad fp16", "plane wgrad bf16", "plane wgrad 2-D", "plane wgrad 3-D",
             "plane wgrad scalar loads", "plane dead tap", "plane empty split", "plane stride 2", "plane dilation",
             "plane time taps", "plane sample boundaries", "plane P = 64k +- 1", "plane P < 64", "bn_apply_plane fp16",
             "bn_apply_plane bf16", "plane bn_apply vector", "plane bn_apply scalar", "plane dropout",
             "plane dropout offset >= 2^32", "plane bn_apply window", "plane padding", "plane padding, vector",
             "plane plane_cstride not a multiple of 64"]


def test_every_entry_point_and_path_is_replayed():
    rows = [r for name in SOURCES for r in run_source(name)]
    counts = {f: sum(f in r["features"] for r in rows) for f in REQUIRED}
    print("\nfeature: launches")
    for f in REQUIRED:
        print(f"  {f:<30s} {counts[f]}")
    wg = sorted((r["res"]["per"], r["res"]["model"], r["res"]["exact"], r["tag"]) for r in rows if r["kind"] == "wgrad")
    print("weight gradients by pixels per split: per, worst model excess, exact error (of max |exact|)")
    for per, m, e, tag in wg:
        print(f"  {per:6d}  {m:.2e}  {e:.2e}  {tag}")
    print("one-plane weight gradients, worst per `per` (of max |model|): fp16 / bf16 (bar wgrad_bar(per))")
    worst = {}
    for r in rows:
        for nm in PLANE_NAMES.values():
            if f"plane wgrad {nm}" in r["features"]:
                k = (r["res"]["per"], nm)
                worst[k] = max(worst.get(k, 0.0), r["res"]["model"])
    for per in sorted({p for p, _ in worst}):
        print(f"  {per:6d}  " + "  ".join(f"{nm} {worst[(per, nm)]:.2e}" if (per, nm) in worst else f"{nm}    -    "
                                          for nm in PLANE_NAMES.values()) + f"  (bar {wgrad_bar(per):.1e})")
    assert all(counts.values()), [f for f, c in counts.items() if not c]
