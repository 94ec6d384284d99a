"""GPU: every launch of the back-to-back kernels (stp3_aspp_fused_fwd: the DeepLab head's ASPP and its 3x3 -> classifier
tail; stp3_block_fused_fwd: the TemporalBlock tails) replayed against the fp64 reference of their contract
(tests/fused_reference.py).

Launches are recorded from the model (dense.aspp_fused / dense.block_tail wrapped while it runs, inputs and bias tables
cloned, what the production call wrote cloned too) at the perceive shape (40 x 56, B = 2) and at the headline 200 x 200
(B = 1, T = 3), and built synthetically for what the model never produces (tests/fused_cases.py).  Each is replayed
twice into sentinel-filled output planes and column sums.  Checked per replay:
  - every stored value within EXACT_BAR of max |exact| (both stages exact, P unsplit);
  - per element against the model (the products the kernel issues and the hi/lo split of P), beyond the 2^-17 split
    allowance of the stored planes, within fused_bar(K);
  - the column sums against the fp64 sums, held to the sum of the magnitudes they add up;
  - every channel outside the written window unchanged; the classifier's padding channels exactly 0;
  - the second launch bitwise equal to the first, and a recorded launch bitwise equal to what production wrote (behind
    its PDL predecessor);
Bias tables differ per image and inputs per sample, so a wrong image or frame is an O(1) error.  The last test asserts
that the replays reached both block layouts and every listed descriptor feature."""
import ast
import ctypes
import inspect
import os
from dataclasses import dataclass
from typing import Optional

import pytest
import torch

from stp3_b200 import _lib, dense
from tests import fused_cases as FC
from tests import fused_reference as FR
from tests import test_conv_contract_gpu as CC

pytestmark = CC.pytestmark
DEV = CC.DEV
EXACT_BAR = CC.EXACT_BAR
SPLIT = CC.SPLIT
SENT = CC.SENT


def fused_bar(K: int) -> float:
    """Model bar of the chained kernels, of max |exact| beyond the split allowance; K = the total reduction length of
    both stages (ASPP: taps x cin_p + 128 per branch; block: 64 per chain tap + 128, + 64 with a projection).  The
    fp32 error of stage 1 reaches the output through P and the stage-2 weights, so the chain could have needed more
    than the single convolution's bar.  Worst measured on an H100 80GB HBM3 (700 W power limit) over every launch of
    this file (table in DESIGN.md section 4): 1.5e-6 at K = 192, 2.3e-6 at K = 896, 6.6e-6 at K = 1280 (the head's
    tail at 200 x 200), 4.4e-6 at K = 2304; block 3.0e-6 at K = 1344, 3.9e-6 at K = 1984.  All lie inside the
    convolution's envelope 5e-7 + 2e-7 sqrt(K) (7.7e-6 at K = 1280), so the bar is the convolution contract's
    model_bar, 4x that envelope."""
    return CC.model_bar(K)


def n_sm() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ recording
def _clone(h: dense.HL) -> dense.HL:
    return dense.HL(h.hi.clone(), h.lo.clone(), h.c)


@dataclass
class AsppCall:
    source: str
    tag: str
    x: dense.HL
    pa: dense.PackedAspp
    img_bias: torch.Tensor
    out_cstride: int
    out_coff: int
    relu: bool
    n_store: int
    prod: Optional[dict] = None          # the window production wrote: {"hi", "lo"}


@dataclass
class BlockCall:
    source: str
    tag: str
    mid: dense.HL
    x: dense.HL
    pb: dense.PackedBlockTail
    hid: torch.Tensor
    img: torch.Tensor
    res: Optional[torch.Tensor]
    out_cstride: int
    col_sums: bool
    prod: Optional[dict] = None          # {"hi", "lo"[, "col_sums"]}


def bare_fused_calls():
    """Calls of aspp_fused / block_tail by their bare names inside dense.py, and imports of them from other modules:
    either would bypass the recorder."""
    names = ("aspp_fused", "block_tail")
    tree = ast.parse(inspect.getsource(dense))
    bare = [n.lineno for n in ast.walk(tree) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and
            n.func.id in names]
    pkg = os.path.dirname(os.path.abspath(dense.__file__))
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                with open(os.path.join(root, f)) as fh:
                    t = ast.parse(fh.read())
                bare += [f"{f}:{n.lineno}" for n in ast.walk(t) if isinstance(n, ast.ImportFrom) and
                         (n.module or "").endswith("dense") and any(a.name in names for a in n.names)]
    return bare


class Recorder:
    def __init__(self, source):
        self.source, self.calls = source, []

    def __enter__(self):
        self.mp = pytest.MonkeyPatch()
        a_orig, b_orig = dense.aspp_fused, dense.block_tail

        def aspp(x, pa, img_bias, out=None, out_coff=0, relu=True, n_store=128, c_out=None):
            y = a_orig(x, pa, img_bias, out=out, out_coff=out_coff, relu=relu, n_store=n_store, c_out=c_out)
            w = slice(out_coff, out_coff + n_store)
            self.calls.append(AsppCall(self.source, "head tail" if not relu else "head aspp", _clone(x), pa,
                                       img_bias.clone(), y.hi.shape[-1], out_coff, relu, n_store,
                                       {"hi": y.hi[..., w].clone(), "lo": y.lo[..., w].clone()}))
            return y

        def block(mid, x, pb, hid_bias, img_bias, res_bias, col_sums=None):
            y = b_orig(mid, x, pb, hid_bias, img_bias, res_bias, col_sums=col_sums)
            prod = {"hi": y.hi.clone(), "lo": y.lo.clone()}
            if col_sums is not None:
                prod["col_sums"] = col_sums.clone()
            self.calls.append(BlockCall(self.source, f"block {len(pb.chains)} chains", _clone(mid), _clone(x), pb,
                                        hid_bias.clone(), img_bias.clone(),
                                        None if res_bias is None else res_bias.clone(), 64, col_sums is not None, prod))
            return y
        self.mp.setattr(dense, "aspp_fused", aspp)
        self.mp.setattr(dense, "block_tail", block)
        return self

    def __exit__(self, *exc):
        self.mp.undo()
        torch.cuda.synchronize()


def rec_perceive():
    """STP3.forward_features, perceive configuration, B = 2 at a 40 x 56 BEV (the conv contract's model)."""
    from stp3_b200.utils import synthetic as syn
    with torch.no_grad():
        model, lcfg = CC._stp3_model(64, 3, [-10.0, 10.0, 0.5], [-14.0, 14.0, 0.5])
        inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
        with Recorder("perceive 40x56") as r:
            model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                   inp["extrinsics"], inp["future_egomotion"])
    return r.calls


def rec_headline():
    """The temporal model of bench.build_model at the headline size: batch 1, 3 frames, 200 x 200."""
    import bench
    with torch.no_grad():
        model = bench.build_model(DEV)
        x = FC.planes(1, 3, 200, 200, 64, 64, seed=31, dev=DEV)
        const = FC.rnd(3, 6, seed=32, scale=0.5, dev=DEV)
        with Recorder("temporal 200x200") as r:
            model.temporal_model.forward_hl(x, const=const)
    return r.calls


# ------------------------------------------------------------------------------------------------ synthetic
def tile_geom(n):
    """(H, W) of one image with exactly n 8 x 16 tiles, both ragged: the largest divisor ty <= 12 of n tile rows"""
    ty = max(d for d in range(1, 13) if n % d == 0)
    return 8 * ty - 3, 16 * (n // ty) - 5


def _aspp(tag, rates, B, T, H, W, *, cin=64, cs=None, n_out=128, n_store=128, relu=True, out_cs=None, out_coff=0,
          seed=0):
    case = FC.aspp_case(cin, rates, n_out=n_out, seed=seed, dev=DEV)
    x = FC.planes(B, T, H, W, cin, cs or cin, seed=seed + 50, dev=DEV)
    ib = FC.rnd(B * T, 128, seed=seed + 51, scale=0.5, dev=DEV)
    if n_out < 128:
        ib[:, n_out:] = 0                     # the classifier's padding rows: exact zeros out
    return AsppCall("synthetic", tag, x, case.pa, ib, out_cs or n_store, out_coff, relu, n_store)


def rec_synthetic_aspp():
    S = n_sm()
    C3 = (3, 3)
    calls = [
        _aspp("1 branch, 1 tap", [None], 1, 1, 21, 37, seed=1),
        _aspp("2 branches, in_cstride > cin, out_coff 16", [None, (2, 2)], 2, 1, 19, 35, cs=128, out_cs=160,
              out_coff=16, seed=2),
        _aspp("4 branches, edge rates", [None, (7, 15), (15, 31), (23, 31)], 1, 1, 48, 64, seed=3),
        _aspp("edge rates 31 / 15, kblocks 2", [(31, 15), None], 1, 1, 64, 48, cin=128, cs=192, seed=4),
        _aspp("rate beyond the map (127)", [None, (127, 127), (40, 3)], 1, 2, 27, 29, seed=5),
        _aspp("tail: no ReLU, n_store 64", [C3], 1, 2, 26, 30, cin=128, n_out=40, n_store=64, relu=False, seed=6),
        _aspp("n_store 64 with ReLU, out_coff 16", [None, C3], 1, 1, 17, 20, n_store=64, out_cs=96, out_coff=16,
              seed=7),
        _aspp("B 2, T 3 (5-D map)", [None, (3, 5)], 2, 3, 13, 22, seed=8),
        _aspp("partial single tile", [None, (1, 1)], 1, 1, 5, 11, seed=9),
        _aspp("1 tile per image, 2 SM + 1 images", [None, (2, 3)], 1, 2 * S + 1, 8, 16, seed=10),
    ]
    for n in (1, S - 1, S, S + 1, 2 * S + 1):
        H, W = tile_geom(n)
        calls.append(_aspp(f"{n} tiles", [None, C3], 1, 1, H, W, seed=20 + n % 7))
    return calls


def _block(tag, layout, proj, B, T, H, W, *, col_sums=True, x_cs=64, out_cs=64, seed=0):
    case = FC.block_case(layout, proj, seed=seed, dev=DEV)
    mid = FC.planes(B, T, H, W, 128, 128, seed=seed + 50, dev=DEV)
    x = FC.planes(B, T, H, W, 64, x_cs, seed=seed + 51, dev=DEV)
    n = B * T
    hid, ib = FC.rnd(n, 128, seed=seed + 52, scale=0.5, dev=DEV), FC.rnd(n, 64, seed=seed + 53, scale=0.5, dev=DEV)
    rb = FC.rnd(n, 64, seed=seed + 54, scale=0.5, dev=DEV) if proj else None
    return BlockCall("synthetic", tag, mid, x, case.pb, hid, ib, rb, out_cs, col_sums)


def rec_synthetic_block():
    S = n_sm()
    calls = []
    for layout, proj in ((0, True), (1, False), (0, False), (1, True)):
        calls += [
            _block(f"L{layout} T 1", layout, proj, 1, 1, 21, 35, seed=1 + layout),
            _block(f"L{layout} B 2 T 3, W = 1 mod 16, H = 1 mod 8", layout, proj, 2, 3, 17, 33, seed=3 + layout),
            _block(f"L{layout} no col_sums, out/x cstride 128", layout, proj, 1, 2, 19, 40, col_sums=False, x_cs=128,
                   out_cs=128, seed=5 + layout),
        ]
    calls.append(_block("L0 col_sums, out cstride 128", 0, True, 2, 2, 9, 17, out_cs=128, seed=7))
    calls.append(_block("L0 1 tile per image, 2 SM + 1 images", 0, True, 1, 2 * S + 1, 8, 16, seed=8))
    calls.append(_block("L1 1 tile per image, 2 SM + 1 images", 1, False, 1, 2 * S + 1, 7, 13, seed=9))
    for n in (1, S - 1, S, S + 1, 2 * S + 1):
        H, W = tile_geom(n)
        calls.append(_block(f"{n} tiles", n % 2, n % 2 == 0, 1, 1, H, W, seed=20 + n % 7))
    return calls


def rec_predict_small(carla):
    """the Prediction model's forward at 40 x 56, B = 2 (tests/test_conv_contract_gpu.py predict_model): the DeepLab
    head of the last SpatialGRU over B x 7 frames"""
    r = Recorder(f"predict {'carla' if carla else 'nuscenes'} 40x56")
    CC.run_predict_small(carla, r)
    return r.calls


def rec_predict_200():
    """STP3._predict_hl on (1, 3, 64, 200, 200) present states: the DeepLab head over 7 frames of 200 x 200"""
    r = Recorder("predict 200x200")
    CC.run_predict_200(r)
    return r.calls


SOURCES = {
    "perceive": rec_perceive,
    "headline": rec_headline,
    "predict_small_nuscenes": lambda: rec_predict_small(False),
    "predict_small_carla": lambda: rec_predict_small(True),
    "predict_200x200": rec_predict_200,
    "synthetic_aspp": rec_synthetic_aspp,
    "synthetic_block": rec_synthetic_block,
}


# ------------------------------------------------------------------------------------------------ replay
def _sent(shape, dtype):
    return torch.full(shape, SENT, dtype=dtype, device=DEV)


def launch_block(c: BlockCall, out: dense.HL, col_sums: Optional[torch.Tensor]):
    """stp3_block_fused_fwd with an output of any channel stride (dense.block_tail always allocates 64 channels)"""
    B, T, H, W, _ = c.x.hi.shape
    d = _lib.BlockDesc()
    d.B, d.T, d.H, d.W = B, T, H, W
    d.mid_cstride, d.x_cstride, d.out_cstride = c.mid.hi.shape[-1], c.x.hi.shape[-1], out.hi.shape[-1]

    def fill(dst, ch):
        src, cin_off, taps, n_mma, tmem_col, k_lo, k_hi = ch
        dst.src, dst.cin_off, dst.n_taps, dst.n_mma, dst.tmem_col, dst.k_lo, dst.k_hi = \
            src, cin_off, len(taps), n_mma, tmem_col, k_lo, k_hi
        for i, t in enumerate(taps):
            dst.taps[i][0], dst.taps[i][1], dst.taps[i][2] = t
    d.n_chain = len(c.pb.chains)
    for i, ch in enumerate(c.pb.chains):
        fill(d.chain[i], ch)
    d.has_res_proj = int(c.pb.res is not None)
    if c.pb.res is not None:
        fill(d.res, c.pb.res)
    for i, v in enumerate(c.pb.piece_col):
        d.piece_col[i] = v
    scratch, nbytes = None, 0
    if col_sums is not None:
        nbytes = _lib.lib().stp3_block_fused_scratch_bytes(B * T)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    ptr = lambda t: t.data_ptr() if t is not None else None          # noqa: E731
    code = _lib.lib().stp3_block_fused_fwd(
        ctypes.byref(d), c.mid.hi.data_ptr(), c.mid.lo.data_ptr(), c.x.hi.data_ptr(), c.x.lo.data_ptr(),
        c.pb.w.data_ptr(), c.hid.data_ptr(), c.img.data_ptr(), ptr(c.res), out.hi.data_ptr(), out.lo.data_ptr(),
        ptr(col_sums), ptr(scratch), nbytes, torch.cuda.current_stream(DEV).cuda_stream)
    _lib.check(code, "stp3_block_fused_fwd")


def _launch(c):
    """one launch into sentinel-filled buffers: {name: tensor}"""
    B, T, H, W, _ = c.x.hi.shape
    shape = (B, T, H, W, c.out_cstride)
    out = dense.HL(_sent(shape, torch.bfloat16), _sent(shape, torch.bfloat16), c.out_cstride)
    bufs = {"hi": out.hi, "lo": out.lo}
    if isinstance(c, AsppCall):
        dense.aspp_fused(c.x, c.pa, c.img_bias, out=out, out_coff=c.out_coff, relu=c.relu, n_store=c.n_store)
    else:
        cs = _sent((B * T, 64), torch.float32) if c.col_sums else None
        launch_block(c, out, cs)
        if cs is not None:
            bufs["col_sums"] = cs
    return bufs


def _window(c):
    return (c.out_coff, c.n_store) if isinstance(c, AsppCall) else (0, 64)


def replay(c):
    first = _launch(c)
    second = _launch(c)
    torch.cuda.synchronize()
    same = all(torch.equal(first[k], second[k]) for k in first)
    c0, n = _window(c)
    keep = torch.ones(c.out_cstride, dtype=torch.bool, device=DEV)
    keep[c0:c0 + n] = False
    untouched = all(bool((first[k][..., keep] == _sent((), torch.bfloat16)).all()) for k in ("hi", "lo"))
    prod = True
    if c.prod is not None:
        prod = all(torch.equal(first[k][..., c0:c0 + n] if k != "col_sums" else first[k], v) for k, v in c.prod.items())
    B, T, H, W, _ = c.x.hi.shape
    got = {"y": (first["hi"][..., c0:c0 + n].double() + first["lo"][..., c0:c0 + n].double()).reshape(B * T, H, W, n)}
    if "col_sums" in first:
        got["col_sums"] = first["col_sums"].double()
    return got, same, untouched, prod, first


def references(c):
    if isinstance(c, AsppCall):
        ref = {m: {"y": FR.aspp(c.x.hi, c.x.lo, c.pa, c.img_bias, n_store=c.n_store, relu=c.relu, model=m)}
               for m in (False, True)}
    else:
        ref = {}
        for m in (False, True):
            y, s = FR.block_tail(c.mid.hi, c.mid.lo, c.x.hi, c.x.lo, c.pb, c.hid, c.img, c.res, model=m)
            ref[m] = {"y": y}
            if c.col_sums:
                ref[m]["col_sums"] = s
    exact, model = ref[False], ref[True]
    scale = {"y": max(float(exact["y"].abs().max()), 1e-20)}
    if "col_sums" in exact:        # a column sum is held to the sum of the magnitudes it adds up
        scale["col_sums"] = max(float(exact["y"].abs().sum(dim=(1, 2)).max()), 1e-20)
    return exact, model, scale


def zero_channels(c) -> list:
    """output channels of an ASPP launch that must be exactly 0: projection rows and per-image biases all zero
    (the classifier's padding rows of the tail instance)"""
    if not isinstance(c, AsppCall):
        return []
    n_br = len(c.pa.taps)
    proj = c.pa.w[-2 * n_br:].float().abs().sum(dim=(0, 1, 3))          # (128,) over blocks, planes, K
    z = (proj == 0) & (c.img_bias.abs().sum(0) == 0)
    return [i for i in range(c.n_store) if bool(z[i])]


def reduction_length(c) -> int:
    if isinstance(c, AsppCall):
        return sum(len(t) for t in c.pa.taps) * c.pa.cin_p + len(c.pa.taps) * 128
    return sum(len(ch[2]) for ch in c.pb.chains) * 64 + 128 + (64 if c.pb.res is not None else 0)


# ------------------------------------------------------------------------------------------------ coverage
def _aspp_sides(c, f):
    """per tap and tile: a side on which the tap window is pure padding (skipped), or overlaps the image by exactly
    one row / column while the neighbouring tile on that side exists and is skipped"""
    _, _, H, W, _ = c.x.hi.shape
    rows, cols = range(0, H, 8), range(0, W, 16)
    for taps in c.pa.taps:
        live_other = []
        for dy, dx in taps:
            for oy in rows:
                if dy < 0 and oy + 7 + dy < 0:
                    f.add("top: skipped")
                if dy < 0 and oy + 7 + dy == 0 and oy >= 8:
                    f.add("top: one row live beside a skipped tile")
                if dy > 0 and oy + dy >= H:
                    f.add("bottom: skipped")
                if dy > 0 and oy + dy == H - 1 and oy + 8 < H:
                    f.add("bottom: one row live beside a skipped tile")
            for ox in cols:
                if dx < 0 and ox + 15 + dx < 0:
                    f.add("left: skipped")
                if dx < 0 and ox + 15 + dx == 0 and ox >= 16:
                    f.add("left: one column live beside a skipped tile")
                if dx > 0 and ox + dx >= W:
                    f.add("right: skipped")
                if dx > 0 and ox + dx == W - 1 and ox + 16 < W:
                    f.add("right: one column live beside a skipped tile")
            if (dy, dx) != (0, 0):
                live_other.append(any(not (oy + 7 + dy < 0 or oy + dy >= H or ox + 15 + dx < 0 or ox + dx >= W)
                                      for oy in rows for ox in cols))
        if live_other and not any(live_other):
            f.add("every non-centre tap skipped")
        if any(abs(v) == 127 for t in taps for v in t):
            f.add("rate 127")


def features(c) -> set:
    B, T, H, W, cs = c.x.hi.shape
    tiles = B * T * -(-H // 8) * -(-W // 16)
    S = n_sm()
    f = {f"source {c.source}"}
    for n, name in ((1, "1"), (S - 1, "SM - 1"), (S, "SM"), (S + 1, "SM + 1"), (2 * S + 1, "2 SM + 1")):
        if tiles == n:
            f.add(f"tiles = {name}")
    if -(-H // 8) * -(-W // 16) == 1 and B * T > S:
        f.add("1 tile per image, more images than SMs")
    if B > 1 and T > 1:
        f.add("B > 1 and T > 1")
    if isinstance(c, AsppCall):
        f.add(f"aspp {len(c.pa.taps)} branches")
        f |= {f"aspp {len(t)}-tap branch" for t in c.pa.taps}
        f.add(f"aspp kblocks {c.pa.cin_p // 64}")
        if cs > c.pa.cin_p:
            f.add("aspp in_cstride > cin")
        f.add(f"aspp n_store {c.n_store}")
        f.add(f"aspp no_relu {int(not c.relu)}")
        if c.out_coff > 0:
            f.add("aspp out_coff > 0")
        if zero_channels(c):
            f.add("aspp zero padding channels")
        if H < 8 and W < 16:
            f.add("aspp one partial tile")
        _aspp_sides(c, f)
    else:
        f.add(f"block layout {0 if len(c.pb.chains) == 3 else 1}")
        f.add("block projection" if c.pb.res is not None else "block identity residual")
        f.add("block col_sums" if c.col_sums else "block no col_sums")
        if T == 1:
            f.add("block T = 1")
        else:
            f.add("block causal tap live")
        if W % 16 == 1:
            f.add("block W = 1 mod 16 (dx = +1 group skipped, dx = 0 live by one column)")
        if H % 8 == 1:
            f.add("block H = 1 mod 8")
        if c.out_cstride > 64:
            f.add("block out_cstride > 64")
        if cs > 64:
            f.add("block x_cstride > 64")
    return f


REQUIRED = (["aspp 1 branches", "aspp 2 branches", "aspp 4 branches", "aspp 1-tap branch", "aspp 9-tap branch",
             "aspp kblocks 1", "aspp kblocks 2", "aspp in_cstride > cin", "aspp n_store 64", "aspp n_store 128",
             "aspp no_relu 0", "aspp no_relu 1", "aspp out_coff > 0", "aspp zero padding channels",
             "aspp one partial tile", "every non-centre tap skipped", "rate 127"] +
            [f"{s}: skipped" for s in ("top", "bottom", "left", "right")] +
            [f"{s}: one {u} live beside a skipped tile" for s, u in (("top", "row"), ("bottom", "row"),
                                                                     ("left", "column"), ("right", "column"))] +
            ["block layout 0", "block layout 1", "block projection", "block identity residual", "block col_sums",
             "block no col_sums", "block T = 1", "block causal tap live",
             "block W = 1 mod 16 (dx = +1 group skipped, dx = 0 live by one column)", "block H = 1 mod 8",
             "block out_cstride > 64", "block x_cstride > 64", "B > 1 and T > 1",
             "1 tile per image, more images than SMs"] +
            [f"tiles = {n}" for n in ("1", "SM - 1", "SM", "SM + 1", "2 SM + 1")])


# ------------------------------------------------------------------------------------------------ driver
_RUNS = {}


def run_source(name):
    if name in _RUNS:
        return _RUNS[name]
    calls = SOURCES[name]()
    assert calls, f"{name}: no fused launch recorded"
    rows = []
    for i, c in enumerate(calls):
        exact, model, scale = references(c)
        got, same, untouched, prod, first = replay(c)
        assert set(got) == set(exact), (set(got), set(exact))
        e_x = max(float((got[k] - exact[k]).abs().max()) / scale[k] for k in got)
        e_m = max(CC._excess(got[k], model[k], SPLIT if k == "y" else 0.0) / scale[k] for k in got)
        zc = zero_channels(c)
        zeros = True
        if zc:
            c0 = _window(c)[0]
            idx = torch.tensor([c0 + z for z in zc], device=DEV)
            zeros = all(bool((first[k].index_select(-1, idx) == 0).all()) for k in ("hi", "lo"))
        K = reduction_length(c)
        kind = "aspp" if isinstance(c, AsppCall) else f"block L{0 if len(c.pb.chains) == 3 else 1}"
        rows.append(dict(call=i, kind=kind, K=K, exact=e_x, model=e_m, bar=fused_bar(K), same=same,
                         untouched=untouched, prod=prod, zeros=zeros, features=features(c),
                         desc=f"{c.tag} {tuple(c.x.hi.shape)}"))
        del exact, model, got, first
    torch.cuda.empty_cache()
    _RUNS[name] = rows
    return rows


def test_no_call_bypasses_the_recorder():
    assert not bare_fused_calls()


@pytest.mark.parametrize("name", list(SOURCES))
def test_fused_launches_against_the_fp64_contract(name):
    rows = run_source(name)
    print(f"\n{name}: {len(rows)} launches")
    for r in rows:
        print(f"  #{r['call']:<3d} {r['kind']:<9s} K {r['K']:<5d} exact {r['exact']:.2e}  model {r['model']:.2e} "
              f"(bar {r['bar']:.1e})  {r['desc']}")
    bad = [(r["call"], r["desc"], r["exact"], r["model"], r["same"], r["untouched"], r["prod"], r["zeros"])
           for r in rows if not (r["exact"] <= EXACT_BAR and r["model"] <= r["bar"] and r["same"] and
                                 r["untouched"] and r["prod"] and r["zeros"])]
    assert not bad, bad


def test_the_model_launches_both_kernels():
    rows = run_source("perceive")
    kinds = [r["kind"] for r in rows]
    assert kinds.count("aspp") == 2 and sum(k.startswith("block") for k in kinds) == 2, kinds


def test_every_layout_and_feature_is_replayed():
    rows = [r for name in SOURCES for r in run_source(name)]
    counts = {f: sum(f in r["features"] for r in rows) for f in REQUIRED}
    worst = {}
    for r in rows:
        w = worst.setdefault(r["kind"], dict(n=0, exact=0.0, model=0.0, K=set()))
        w["n"] += 1
        w["exact"], w["model"] = max(w["exact"], r["exact"]), max(w["model"], r["model"])
        w["K"].add(r["K"])
    print("\nkernel: launches, worst exact / model error (of max |exact|), reduction lengths")
    for k, w in sorted(worst.items()):
        print(f"  {k:<9s} {w['n']:3d}  {w['exact']:.2e} / {w['model']:.2e}  K {sorted(w['K'])}")
    print("feature: launches")
    for f in REQUIRED:
        print(f"  {f:<72s} {counts[f]}")
    assert {"aspp", "block L0", "block L1"} <= set(worst), set(worst)
    assert all(counts.values()), [f for f, c in counts.items() if not c]
