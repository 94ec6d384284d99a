"""GPU: every convolution the model launches, replayed under every tiling the autotuner may pick, against a float64
reference of the stp3_conv_fwd contract (tests/conv_reference.py).

The calls are recorded from the model itself (dense.conv wrapped while the forward / backward runs), so the descriptors
are the production ones: frame windows, trimmed K ranges, channel windows of concat tensors, split 256-column launches,
output-size overrides of the input-gradient phases, fused heads, column sums.  The Prediction model adds K windows that
start inside a buffer (cin_off 64 of the conv-GRU cell and of the Bottleblock's second 7 x 7 launch), 49-tap layers and
the decoder over 7 frames
(predict_model at 40 x 56 with both gate sets, and each distinct convolution of _predict_hl at 200 x 200).  The
trainable trunk's train steps (tests/test_train_contract_gpu.py trunk_step) add the expand convolutions' 256-column
chunks, the projections and their input gradients in 256-channel chunks, at channel counts that are not multiples of
64; at 224 x 480 only one call per descriptor is replayed under every tiling, the repeats under (0, 0).  Each
recorded call is replayed with
tune = (0, 0) (the kernel's own heuristics: graph capture, STP3_CONV_AUTOTUNE=0) and with every candidate of
dense.tune_candidates, into outputs pre-filled with a sentinel.  Checked per replay:
  - every written value against the exact fp64 convolution (the project's 3e-5 of max bar) and against the fp64
    evaluation of the three bf16 products the kernel issues, element by element up to the rounding of the stored
    hi/lo planes, with a bar measured on the H100 that grows with the reduction length (see model_bar);
  - nothing outside the written channel windows changed;
  - a second launch of the same tiling is bitwise identical (column sums included).
Descriptor features the model never produces are covered by a few synthetic calls; the last test asserts that the
replays reached every kernel instantiation and every feature, with the instantiation, column-block width, stacked
operand and resident / streamed weights the library reports for the call (stp3_conv_tiling_op).

One-plane convolutions (stp3_conv_fwd_plane, the forward and input-gradient convolutions of a train step under
torch.autocast): the same four train-mode modules (tests/test_train_contract_gpu.py *_step) run one step in float16
and in bfloat16, plus synthetic plane calls for a front-trimmed K range at 128 columns with a stride-2 sigmoid NCHW output, causal taps
at frame 0, a 256-column layer and input-gradient phases of unequal sizes.  The fp64 tap sum of the plane values is
both the exact result and the one-product model.  Checked per replay, besides the window and repeatability checks:
every element within model_bar(K) of max |model| and within CONV_ULPS fp32 ulps of the summed magnitudes of its terms;
the fp32 output's guard untouched; the replay of the tiling production forced bitwise equal to what it wrote; every
+8 tiling bitwise equal to the same tiling without +8 (the stacked operand does not apply to a plane)."""
import ast
import inspect
import os
import time
from dataclasses import dataclass
from typing import Optional

import pytest
import torch

from stp3_b200 import dense
from tests import conv_reference as R
from tests import test_train_contract_gpu as TC

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif("STP3_CONV_GROUP" in os.environ,
                                 reason="STP3_CONV_GROUP overrides the tiling of every launch (read once per process)")]
DEV = "cuda:0"
EXACT_BAR = 3e-5      # of max |exact|: bf16x3 products with fp32 accumulation (as in test_conv_gpu.py)
SENT = -1.5e30        # sentinel of every output buffer before a replay
GUARD = 64            # sentinel elements behind every fp32 output
CONV_ULPS = 64        # one-plane bar in fp32 ulps of the summed magnitudes (tests/test_amp_contract_gpu.py)
ULP = 2.0 ** -23
PLANE_NAMES = {torch.float16: "fp16", torch.bfloat16: "bf16"}


# Against the three-product model the kernel may differ by two things only:
#  - the hi/lo split of a stored output: hi = bf16(v) leaves |v - hi| <= 2^-9 |v| and lo = bf16(v - hi) rounds that by
#    at most 2^-9 of itself, so hi + lo is within 2^-18 |v| of the kernel's fp32 value v.  SPLIT allows twice that,
#    per element (v itself differs from the model by the accumulation term below); it is zero for the fp32, head and
#    column-sum outputs;
#  - fp32 accumulation and the fp32 epilogue, held to model_bar(K) of max |exact| beyond the split allowance,
#    K = taps x input channels.  Worst measured on an H100 80GB HBM3 (700 W power limit) over every recorded layer and
#    tiling (table in DESIGN.md section 4): 4.8e-7 at K = 64, 4.0e-6 at K = 576, 9.5e-6 at K = 2304, 1.1e-5 at
#    K = 3136, all below 5e-7 + 2e-7 sqrt(K).  The bar is 4x that envelope: 8.4e-6 at K = 64 and 2.1e-5 at K = 576,
#    where losing the hi.lo products of one 16-channel K step moves an output by up to 16/576 * 2^-9 = 5.4e-5 of its
#    magnitude.  Up to K ~ 1200 it is tighter than EXACT_BAR; above, EXACT_BAR is the binding one.
SPLIT = 2.0 ** -17


def model_bar(K: int) -> float:
    return 4 * (5e-7 + 2e-7 * K ** 0.5)


# ------------------------------------------------------------------------------------------------ recording
@dataclass
class Call:
    source: str
    x: dense.HL
    pc: dense.PackedConv
    kw: dict                                  # dense.conv keywords; output tensors replaced by their specs
    tag: str = ""
    prod: Optional[tuple] = None              # one-plane calls: (tiling production forced, its out_f32)
    chunk: Optional[tuple] = None             # trunk calls: (dense_train function, chunk index, chunks in the call)
    all_tilings: bool = True                  # False: replayed under (0, 0) only (a repeat of a replayed descriptor)

    @property
    def plane(self):
        return self.x.hi.dtype if self.x.lo is None else None


def _clone_hl(h: Optional[dense.HL]):
    return None if h is None else dense.HL(h.hi.clone(), h.lo.clone() if h.lo is not None else None, h.c)


def record(source: str, x: dense.HL, pc: dense.PackedConv, kw: dict, tag: str = "") -> Call:
    """Clone the inputs of a dense.conv call; outputs are kept as specs (shape, window) and re-created per replay."""
    kw = dict(kw)
    kw.pop("tune", None)
    store = kw.pop("store", True)
    B, Tt, H, W, _ = x.hi.shape
    T = kw["frames"][1] if kw.get("frames") is not None else Tt
    s = pc.stride
    Ho, Wo = kw["out_hw"] if kw.get("out_hw") is not None else ((H + s - 1) // s, (W + s - 1) // s)
    rec = {k: v for k, v in kw.items() if not isinstance(v, (torch.Tensor, dense.HL, dict))}
    rec["residual"] = _clone_hl(kw.get("residual"))
    rec["img_bias"] = kw["img_bias"].clone() if kw.get("img_bias") is not None else None
    for k in ("out", "out2"):
        rec[k] = tuple(kw[k].hi.shape) if kw.get(k) is not None else None
    if rec["out"] is None and kw.get("out_f32") is None and store:
        rec["out"] = (B, T, Ho, Wo, pc.bn)
    rec["out_f32"] = tuple(kw["out_f32"].shape) if kw.get("out_f32") is not None else None
    rec["col_sums"] = tuple(kw["col_sums"].shape) if kw.get("col_sums") is not None else None
    if kw.get("head") is not None:
        hd = kw["head"]
        tensors = []
        outs = []
        for t, ch in hd["outs"]:
            i = next((j for j, u in enumerate(tensors) if u is t), None)
            if i is None:
                tensors.append(t)
                i = len(tensors) - 1
            outs.append((i, ch))
        rec["head"] = {"w": hd["w"].clone(), "b": hd["b"].clone(), "sigmoid_mask": int(hd.get("sigmoid_mask", 0)),
                       "outs": outs, "shapes": [tuple(t.shape) for t in tensors]}
    else:
        rec["head"] = None
    rec["geom"] = (B, Tt, T, H, W, Ho, Wo)
    return Call(source, _clone_hl(x), pc, rec, tag)


def bare_conv_calls():
    """Calls of `conv` by its bare name inside stp3_b200/dense.py, and imports of it from other modules: either would
    bypass a wrapper installed on dense.conv."""
    tree = ast.parse(inspect.getsource(dense))
    bare = [n.lineno for n in ast.walk(tree) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id == "conv"]
    pkg = os.path.dirname(os.path.abspath(dense.__file__))
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                with open(os.path.join(root, f)) as fh:
                    t = ast.parse(fh.read())
                bare += [f"{f}:{n.lineno}" for n in ast.walk(t) if isinstance(n, ast.ImportFrom) and
                         (n.module or "").endswith("dense") and any(a.name == "conv" for a in n.names)]
    return bare


class Recorder:
    """One-plane calls also keep what production wrote with the tiling it forced (the train path passes tune)."""
    def __init__(self, source):
        self.source, self.calls = source, []

    def __enter__(self):
        self.mp = pytest.MonkeyPatch()
        orig = dense.conv

        def wrapper(x, pc, **kw):
            call = record(self.source, x, pc, kw)
            self.calls.append(call)
            out = orig(x, pc, **kw)
            if x.lo is None and kw.get("tune") is not None:
                call.prod = (tuple(kw["tune"]), kw["out_f32"].clone())
            return out
        self.mp.setattr(dense, "conv", wrapper)
        return self

    def __exit__(self, *exc):
        self.mp.undo()
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ the model's calls
def _stp3_model(C, S, xb, yb):
    from oracle import torch_dense as TD
    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    from stp3_b200.utils import geometry as G
    from stp3_b200.utils import synthetic as syn
    cfg = get_cfg({"LIFT": {"X_BOUND": xb, "Y_BOUND": yb, "D_BOUND": [2.0, 10.0, 1.0]}, "IMAGE": {"FINAL_DIM": (32, 48)},
                   "TIME_RECEPTIVE_FIELD": S, "MODEL": {"ENCODER": {"OUT_CHANNELS": C}}})
    lcfg = syn.LiftSplatConfig(x_bound=tuple(xb), y_bound=tuple(yb), d_bound=(2.0, 10.0, 1.0), final_dim=(32, 48),
                               out_channels=C, n_cameras=2, receptive_field=S)
    model = TD.init_exact(STP3(cfg, backbone=torch.nn.Identity()), seed=7).eval()
    model.frustum.copy_(model.create_frustum())
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
    model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
    return model.to(DEV), lcfg


def rec_perceive(block_fused):
    """STP3.forward_features, perceive configuration, B = 2 at a 40 x 56 BEV: ragged 8 x 16 tiles at every decoder level
    (the decoder's skip additions need multiples of 8) and 5 x 7 at the deepest one."""
    from stp3_b200.utils import synthetic as syn
    mp = pytest.MonkeyPatch()
    mp.setenv("STP3_BLOCK_FUSED", block_fused)
    try:
        with torch.no_grad():
            model, lcfg = _stp3_model(64, 3, [-10.0, 10.0, 0.5], [-14.0, 14.0, 0.5])
            inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
            with Recorder(f"perceive fused={block_fused}") as r:
                model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                       inp["extrinsics"], inp["future_egomotion"])
    finally:
        mp.undo()
    return r.calls


def rec_stress():
    """The stress shape: C = 128 context channels, receptive field S = 5 (four temporal blocks, 134-channel input)."""
    from stp3_b200.utils import synthetic as syn
    with torch.no_grad():
        model, lcfg = _stp3_model(128, 5, [-8.0, 8.0, 0.5], [-8.0, 8.0, 0.5])
        inp = syn.lift_inputs(lcfg, 1, seed=5, random_pose=True)
        with Recorder("stress C128 S5") as r:
            model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                   inp["extrinsics"], inp["future_egomotion"])
    return r.calls


def predict_model(carla):
    """The Prediction model (PROBABILISTIC on, four future frames) with the gate set of nuScenes (instance heads over
    the 7 frames) or CARLA (pedestrian and hdmap; hdmap reads the present frame, a one-frame window at frame 2 of 7),
    at a 40 x 56 BEV, built like tests/test_predict_gpu.py's model: the distribution goes 40 x 56 -> 20 x 28 -> 10 x 14
    -> 5 x 7 -> 3 x 4."""
    from oracle.make_golden_predict import build_prediction_model, predict_cfg
    from stp3_b200.utils import synthetic as syn
    xb, yb = [-10.0, 10.0, 0.5], [-14.0, 14.0, 0.5]
    cfg = predict_cfg(carla)
    cfg.merge({"LIFT": {"X_BOUND": xb, "Y_BOUND": yb, "D_BOUND": [2.0, 10.0, 1.0]}, "IMAGE": {"FINAL_DIM": (32, 48)}})
    lcfg = syn.LiftSplatConfig(x_bound=tuple(xb), y_bound=tuple(yb), d_bound=(2.0, 10.0, 1.0), final_dim=(32, 48),
                               out_channels=64, n_cameras=2, receptive_field=cfg.TIME_RECEPTIVE_FIELD)
    return build_prediction_model(cfg).to(DEV), lcfg


def run_predict_small(carla, recorder):
    """STP3.forward_features of predict_model(carla) on B = 2 synthetic samples inside `recorder` (a context manager);
    returns the outputs"""
    from stp3_b200.utils import synthetic as syn
    with torch.no_grad():
        model, lcfg = predict_model(carla)
        inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
        with recorder:
            return model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                          inp["extrinsics"], inp["future_egomotion"])


def run_predict_200(recorder):
    """STP3._predict_hl on (1, 3, 64, 200, 200) present states (the headline rig's BEV; the distribution ends 25 -> 13)
    inside `recorder`"""
    from oracle.make_golden_predict import build_prediction_model, predict_cfg
    from stp3_b200.utils import synthetic as syn
    with torch.no_grad():
        model = build_prediction_model(predict_cfg(False)).to(DEV)
        s = syn.exact_gauss((1, 3, 64, 200, 200), torch.Generator().manual_seed(12)).to(DEV)
        states = dense.from_f32(s)
        with recorder:
            return model._predict_hl(states)


def _distinct(calls):
    """one call per descriptor (packed convolution, keywords and geometry): the Dual_GRU's steps repeat theirs"""
    seen, out = set(), []
    for c in calls:
        key = (id(c.pc), repr(sorted((k, v) for k, v in c.kw.items() if k not in ("residual", "img_bias", "head"))),
               c.x.hi.shape, c.kw["residual"] is not None)
        if key not in seen:
            seen.add(key)
            out.append(c)
    return out


def rec_predict_small(carla):
    r = Recorder(f"predict {'carla' if carla else 'nuscenes'} 40x56")
    run_predict_small(carla, r)
    return r.calls


def rec_predict_200():
    r = Recorder("predict 200x200")
    run_predict_200(r)
    return _distinct(r.calls)


def rec_encoder_heads():
    """Encoder.heads_hl at the shape of test_encoder_heads_vs_reference_golden: DeepLabHead(160 -> 160, hidden 64) +
    UpsamplingConcat(216 -> 64 / 48) for the context features and the depth logits."""
    from oracle import torch_dense as TD
    from oracle.make_golden_dense import dense_input
    from stp3_b200.config import get_cfg
    from stp3_b200.models.encoder import Encoder
    with torch.no_grad():
        enc = TD.init_exact(Encoder(get_cfg().MODEL.ENCODER, D=48, backbone=torch.nn.Identity()), seed=11).eval().to(DEV)
        r_hi, r_lo = dense_input((2, 160, 14, 30), 21).to(DEV), dense_input((2, 56, 28, 60), 22).to(DEV)
        with Recorder("encoder heads") as r:
            enc.heads_hl(r_lo, r_hi)
    return r.calls


def rec_decoder_train():
    """One train-mode decoder step (batch-statistics BatchNorm): forward convolutions (conv_raw) and the input
    gradients (conv_dgrad: stride-1 and stride-2 phase convolutions) at 40 x 56 -> 20 x 28 -> 10 x 14 -> 5 x 7."""
    from oracle import torch_dense as TD
    from oracle.make_golden_dense import GATES_PERCEIVE
    from stp3_b200.models.decoder import Decoder
    dec = TD.init_exact(Decoder(64, 2, 3, 2, GATES_PERCEIVE), seed=2).train().to(DEV)
    g = torch.Generator().manual_seed(6)
    x = (torch.randn(1, 3, 64, 40, 56, generator=g)).to(DEV).requires_grad_(True)
    with Recorder("decoder train") as r:
        out = dec(x)
        loss = sum((v * torch.randn(v.shape, generator=g).to(DEV)).sum() for v in out.values() if v is not None)
        loss.backward()
    return r.calls


def rec_decoder_full():
    """The decoder of bench.build_model at the headline size: batch 1, 3 frames, 200 x 200 BEV."""
    import bench
    with torch.no_grad():
        model = bench.build_model(DEV)
        g = torch.Generator().manual_seed(8)
        x = torch.randn(1, 3, 64, 200, 200, generator=g).to(DEV)
        with Recorder("decoder 200x200") as r:
            model.decoder(x)
    return r.calls


TRUNK_CONVS = ("conv_raw", "conv1x1_raw", "conv1x1_dgrad", "conv_dgrad")


def rec_trunk(name):
    """One train step of the trainable trunk (tests/test_train_contract_gpu.py trunk_step): the expand convolutions in
    chunks of at most 256 columns (conv1x1_raw), the projections (conv_raw), their input gradients in chunks of at most
    256 input channels (conv1x1_dgrad) and the expand convolutions' input gradients (conv_dgrad).  Each call is marked
    with the dense_train function that made it and its chunk.  At 224 x 480 only the first call of each descriptor is
    replayed under every tiling, the others under (0, 0)."""
    from stp3_b200 import dense_train
    r = Recorder(f"trunk train {name}")
    mp = pytest.MonkeyPatch()

    def marked(fn_name, fn):
        def f(*a, **kw):
            i0 = len(r.calls)
            out = fn(*a, **kw)
            new = r.calls[i0:]
            for j, c in enumerate(new):          # the outermost function marks last: conv1x1_raw over its conv_raw
                c.chunk = (fn_name, j, len(new))
            return out
        return f
    for fn_name in TRUNK_CONVS:
        mp.setattr(dense_train, fn_name, marked(fn_name, getattr(dense_train, fn_name)))
    try:
        with r:
            TC.trunk_step(*TC.TRUNK_STEPS[name])
    finally:
        mp.undo()
    assert all(c.chunk is not None for c in r.calls), "a trunk convolution outside the marked dense_train functions"
    if name.endswith("224x480"):
        seen = set()
        for c in r.calls:
            key = (tuple(c.pc.taps), c.pc.cin_p, c.pc.bn, c.pc.cout, c.pc.stride, c.pc.k_lo, c.pc.k_hi, c.x.hi.shape,
                   c.x.c, repr(sorted((k, v) for k, v in c.kw.items() if k not in ("residual", "img_bias", "head"))))
            c.all_tilings = key not in seen
            seen.add(key)
    return r.calls


def _rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(*shape, generator=g) * 2 - 1) * scale).to(DEV)


def _hl(B, T, H, W, c, cp, seed):
    x = torch.zeros(B, T, H, W, cp, device=DEV)
    x[..., :c] = _rnd(B, T, H, W, c, seed=seed)
    hi, lo = dense.split_hilo(x)
    return dense.HL(hi, lo, c)


def rec_synthetic():
    """Descriptors the model does not produce (or may stop producing): 8-mod-16 output and residual windows (scalar
    stores), a front-trimmed K range at 128 columns, a partial window of a 256-column layer with a ragged channels-last
    fp32 output, frame windows with column sums and a sigmoid NCHW output, a stride-2 fused head, two destinations,
    input-gradient phases of unequal sizes."""
    calls = []
    # 64 columns, 35 input channels (K trimmed at the back), scalar output and residual stores
    pc = dense.pack_conv(_rnd(40, 35, 3, 3, seed=1, scale=0.1), _rnd(40, seed=2))
    calls.append(record("synthetic", _hl(1, 2, 19, 21, 35, 64, 3), pc,
                        dict(out=dense.HL.empty(1, 2, 19, 21, 80, DEV, cp=80), out_coff=8, n_store=40, relu=True,
                             residual=_hl(1, 2, 19, 21, 72, 72, 4), res_coff=8), "scalar stores"))
    # 128 columns (112 carry weights), K range trimmed at the front, residual after the activation, per-image bias
    pc = dense.pack_conv(_rnd(100, 40, 3, 3, seed=5, scale=0.1), _rnd(100, seed=6), in_layout=[(0, 40, 24)], cin_p=64)
    assert pc.k_lo == 16 and pc.bn == 128
    calls.append(record("synthetic", _hl(2, 1, 23, 35, 64, 64, 7), pc,
                        dict(relu=True, residual=_hl(2, 1, 23, 35, 128, 128, 8), res_after_act=True,
                             img_bias=_rnd(2, 128, seed=9)), "k_lo > 0"))
    # 256 columns as two launches, 200 stored, channels-last fp32 output of 13 channels
    pc = dense.pack_conv(_rnd(256, 64, 3, 3, seed=10, scale=0.05), _rnd(256, seed=11))
    calls.append(record("synthetic", _hl(1, 2, 17, 30, 64, 64, 12), pc,
                        dict(out=dense.HL.empty(1, 2, 17, 30, 256, DEV, cp=256), n_store=200,
                             out_f32=torch.empty(2, 17, 30, 13, device=DEV), n_valid=13, out_f32_nhwc=True), "bn 256"))
    # causal (2, 3, 3) over frames [1, 3) of 3, column sums, sigmoid fp32 NCHW output
    pc = dense.pack_conv(_rnd(64, 64, 2, 3, 3, seed=13, scale=0.05), _rnd(64, seed=14))
    calls.append(record("synthetic", _hl(2, 3, 21, 18, 64, 64, 15), pc,
                        dict(frames=(1, 2), relu=True, col_sums=torch.empty(4, 64, device=DEV),
                             out_f32=torch.empty(4, 5, 21, 18, device=DEV), n_valid=5, sigmoid=True), "frames"))
    # stride 2, 128 columns, fused 1x1 head (three outputs, one with a sigmoid), nothing stored
    pc = dense.pack_conv(_rnd(128, 64, 3, 3, seed=16, scale=0.05), _rnd(128, seed=17), stride=2)
    oa, ob = torch.empty(2, 2, 13, 9, device=DEV), torch.empty(2, 1, 13, 9, device=DEV)
    calls.append(record("synthetic", _hl(1, 2, 25, 17, 64, 64, 18), pc,
                        dict(relu=True, store=False, head={"w": _rnd(3, 128, seed=19, scale=0.1), "b": _rnd(3, seed=20),
                                                            "outs": [(oa, 0), (oa, 1), (ob, 0)], "sigmoid_mask": 4}),
                        "head"))
    # two destinations: columns [0, 48) into a concat tensor at channel 40, [64, 128) into a second tensor
    pc = dense.pack_conv(_rnd(128, 64, 1, 1, seed=21, scale=0.1), _rnd(128, seed=22))
    calls.append(record("synthetic", _hl(2, 1, 21, 35, 64, 64, 23), pc,
                        dict(out=dense.HL.empty(2, 1, 21, 35, 128, DEV, cp=128), out_coff=40, n_store=48, relu=True,
                             out2=dense.HL.empty(2, 1, 21, 35, 64, DEV, cp=64), n_store2=64, relu2=False,
                             img_bias=_rnd(2, 128, seed=24)), "out2"))
    # input gradient of a 3x3 stride-2 convolution of a 9 x 7 image: four phase convolutions of the 5 x 4 output
    # gradient with unequal output sizes (5 x 4, 5 x 3, 4 x 4, 4 x 3) -- the model's decoder sizes are all even
    from stp3_b200 import dense_train
    H, W = 9, 7
    g = _hl(2, 1, 5, 4, 64, 64, 25)
    for (py, px), pc in dense_train.pack_dgrad(_rnd(64, 40, 3, 3, seed=26, scale=0.1), 2, 1):
        Hp, Wp = (H - py + 1) // 2, (W - px + 1) // 2
        calls.append(record("synthetic", g, pc,
                            dict(out_f32=torch.empty(2, Hp, Wp, 40, device=DEV), n_valid=40, out_f32_nhwc=True,
                                 out_hw=(Hp, Wp), store=False), f"dgrad phase {py}{px}"))
    return calls


def rec_amp(mode, step, *args):
    """one step of a train-mode module (tests/test_train_contract_gpu.py <step>) with its forward under
    torch.autocast(dtype=mode): the one-plane convolutions of the forward and of the input gradients"""
    with Recorder(f"{step} {args} {PLANE_NAMES[mode]}") as r:
        getattr(TC, step)(*args, mode=mode)
    calls = [c for c in r.calls if c.plane == mode]
    assert len(calls) == len(r.calls), "a hi/lo convolution inside an autocast step"
    return calls


def _plane(B, T, H, W, c, cp, seed, mode):
    x = torch.zeros(B, T, H, W, cp, dtype=mode, device=DEV)
    x[..., :c] = _rnd(B, T, H, W, c, seed=seed, scale=2.0).to(mode)
    return dense.HL(x, None, c)


def rec_synthetic_plane(mode):
    """One-plane calls the modules may not produce: a 128-column layer with a front-trimmed K range, stride 2 and a
    sigmoid NCHW output of 7 channels; 40 output channels of 64 with a trimmed K range, a per-image bias and a
    channels-last output; causal (2, 3, 3) taps over frames [0, 2) of 3 (the causal taps of frame 0 read nothing);
    256 columns (two column blocks) of 200 channels; 1x1 layers of 128 columns with resident weights, K full and
    trimmed; the input-gradient phases of a 3x3 stride-2 convolution of a 9 x 7
    image (output sizes 5 x 4, 5 x 3, 4 x 4, 4 x 3)."""
    from stp3_b200 import dense_train
    calls = []

    def add(x, pc, tag, **kw):
        calls.append(record(f"synthetic {PLANE_NAMES[mode]}", x, pc, dict(kw, store=False), tag))
    pc = dense.pack_conv(_rnd(100, 40, 3, 3, seed=31, scale=0.1), _rnd(100, seed=32), in_layout=[(0, 40, 24)], cin_p=64,
                         stride=2, plane=mode)
    assert pc.k_lo == 16 and pc.bn == 128
    add(_plane(2, 1, 23, 35, 64, 64, 33, mode), pc, "k_lo > 0, stride 2, sigmoid", relu=False,
        out_f32=torch.empty(2, 7, 12, 18, device=DEV), n_valid=7, sigmoid=True)
    pc = dense.pack_conv(_rnd(40, 35, 3, 3, seed=34, scale=0.1), _rnd(40, seed=35), plane=mode)
    add(_plane(1, 2, 19, 21, 35, 64, 36, mode), pc, "n_mma < bn, img_bias", relu=True, img_bias=_rnd(2, 64, seed=37),
        out_f32=torch.empty(2, 19, 21, 40, device=DEV), n_valid=40, out_f32_nhwc=True)
    pc = dense.pack_conv(_rnd(64, 64, 2, 3, 3, seed=38, scale=0.05), _rnd(64, seed=39), plane=mode)
    add(_plane(2, 3, 21, 18, 64, 64, 40, mode), pc, "causal frames [0, 2)", frames=(0, 2), relu=True,
        out_f32=torch.empty(4, 5, 21, 18, device=DEV), n_valid=5, sigmoid=True)
    pc = dense.pack_conv(_rnd(200, 128, 3, 3, seed=41, scale=0.05), _rnd(200, seed=42), plane=mode)
    add(_plane(1, 2, 17, 30, 128, 128, 43, mode), pc, "bn 256",
        out_f32=torch.empty(2, 17, 30, 200, device=DEV), n_valid=200, out_f32_nhwc=True)
    for cin in (35, 64):      # 1x1 at 128 columns: weights resident, full and trimmed K
        pc = dense.pack_conv(_rnd(100, cin, 1, 1, seed=46 + cin, scale=0.1), _rnd(100, seed=47), plane=mode)
        add(_plane(2, 1, 13, 22, cin, 64, 48, mode), pc, f"1x1 cin {cin} -> 128 columns", relu=True,
            out_f32=torch.empty(2, 13, 22, 100, device=DEV), n_valid=100, out_f32_nhwc=True)
    H, W = 9, 7
    g = _plane(2, 1, 5, 4, 64, 64, 44, mode)
    for (py, px), pc in dense_train.pack_dgrad(_rnd(64, 40, 3, 3, seed=45, scale=0.1), 2, 1, plane=mode):
        Hp, Wp = (H - py + 1) // 2, (W - px + 1) // 2
        add(g, pc, f"dgrad phase {py}{px}", out_f32=torch.empty(2, Hp, Wp, 40, device=DEV), n_valid=40,
            out_f32_nhwc=True, out_hw=(Hp, Wp))
    return calls


AMP_STEPS = {   # name: (step, args) -- small maps, as the fp32 train sources
    "decoder": ("decoder_step", ((1, 3, 64, 32, 48), TC.GATES_ALL)),
    "deeplab_temporal": ("deeplab_step", (64, 64, 128, 2, 24, 32)),
    "deeplab_encoder": ("deeplab_step", (160, 160, 64, 2, 14, 30)),
    "temporal": ("temporal_step", (70, 6, 3, 2, 24, 32)),
    "encoder_heads_feat": ("encoder_heads_step", ("feat",)),
    "encoder_heads_uc": ("encoder_heads_step", ("uc",)),
}

SOURCES = {
    "perceive_fused": lambda: rec_perceive("1"),
    "perceive_unfused": lambda: rec_perceive("0"),
    "stress": rec_stress,
    "encoder_heads": rec_encoder_heads,
    "decoder_train": rec_decoder_train,
    "decoder_full": rec_decoder_full,
    "predict_small_nuscenes": lambda: rec_predict_small(False),
    "predict_small_carla": lambda: rec_predict_small(True),
    "predict_200x200": rec_predict_200,
    "synthetic": rec_synthetic,
}
SOURCES.update({_nm: (lambda n=_nm: rec_trunk(n)) for _nm in TC.TRUNK_STEPS})
for _m in PLANE_NAMES:
    SOURCES.update({f"amp_{nm}_{PLANE_NAMES[_m]}": (lambda m=_m, st=st, a=a: rec_amp(m, st, *a))
                    for nm, (st, a) in AMP_STEPS.items()})
    SOURCES[f"synthetic_plane_{PLANE_NAMES[_m]}"] = lambda m=_m: rec_synthetic_plane(m)


# ------------------------------------------------------------------------------------------------ replay
def _sentinel(dtype):
    return torch.tensor(SENT, dtype=dtype, device=DEV)


def _buffers(call: Call):
    """Fresh output tensors filled with the sentinel, and the dense.conv keywords that use them."""
    kw = {k: v for k, v in call.kw.items() if k not in ("out", "out2", "out_f32", "col_sums", "head", "geom")}
    kw["store"] = call.kw["out"] is not None
    bufs = {}

    def sent(shape, dtype):
        return torch.full(shape, SENT, dtype=dtype, device=DEV)
    for k in ("out", "out2"):
        if call.kw[k] is not None:
            shape = call.kw[k]
            kw[k] = dense.HL(sent(shape, torch.bfloat16), sent(shape, torch.bfloat16), shape[-1])
            bufs[k + ".hi"], bufs[k + ".lo"] = kw[k].hi, kw[k].lo
    if call.kw["out_f32"] is not None:
        shape = call.kw["out_f32"]
        n = int(torch.Size(shape).numel())
        store = sent((n + GUARD,), torch.float32)
        kw["out_f32"] = bufs["out_f32"] = store[:n].view(shape)
        bufs["out_f32.guard"] = store[n:]
    if call.kw["col_sums"] is not None:
        kw["col_sums"] = bufs["col_sums"] = sent(call.kw["col_sums"], torch.float32)
    hd = call.kw["head"]
    if hd is not None:
        tensors = [sent(s, torch.float32) for s in hd["shapes"]]
        kw["head"] = {"w": hd["w"], "b": hd["b"], "sigmoid_mask": hd["sigmoid_mask"],
                      "outs": [(tensors[i], ch) for i, ch in hd["outs"]]}
        for i, t in enumerate(tensors):
            bufs[f"head.t{i}"] = t
    return kw, bufs


def _written(call: Call, kw: dict, bufs: dict):
    """(values written by the call as float64 {name: tensor} laid out like R.epilogue, {buffer: mask of the elements
    the call must leave untouched})"""
    B, Tt, T, H, W, Ho, Wo = call.kw["geom"]
    bn = call.pc.bn
    got, keep = {}, {}
    for k, coff_k, n_k, default in (("out", "out_coff", "n_store", bn), ("out2", "out2_coff", "n_store2", 64)):
        if k in kw:
            h = kw[k]
            c0, n = call.kw.get(coff_k, 0), call.kw.get(n_k, 0) or default
            got["y" if k == "out" else "y2"] = R.join(h)[..., c0:c0 + n].reshape(B * T, Ho, Wo, n)
            m = torch.ones(h.hi.shape[-1], dtype=torch.bool, device=DEV)
            m[c0:c0 + n] = False
            keep[k + ".hi"] = keep[k + ".lo"] = m
    if "out_f32" in kw:
        got["f32"] = kw["out_f32"].double()
        keep["out_f32.guard"] = torch.ones(GUARD, dtype=torch.bool, device=DEV)
    if "col_sums" in kw:
        got["col_sums"] = kw["col_sums"].double()
    if "head" in kw:
        hd = call.kw["head"]
        for k, (i, ch) in enumerate(hd["outs"]):
            got[f"head{k}"] = bufs[f"head.t{i}"][:, ch].double()
        for i, shape in enumerate(hd["shapes"]):
            m = torch.ones(shape[1], dtype=torch.bool, device=DEV)
            for j, ch in hd["outs"]:
                if j == i:
                    m[ch] = False
            keep[f"head.t{i}"] = m.view(1, -1, 1, 1).expand(shape)
    return got, keep


def replay(call: Call, cfg):
    """(values written, two launches bitwise equal, nothing outside the windows changed)"""
    return _replay(call, cfg)[:3]


def _replay(call: Call, cfg):
    kw, bufs = _buffers(call)
    dense.conv(call.x, call.pc, tune=cfg, **kw)
    first = {k: t.clone() for k, t in bufs.items()}
    kw2, bufs2 = _buffers(call)
    dense.conv(call.x, call.pc, tune=cfg, **kw2)
    torch.cuda.synchronize()
    same = all(torch.equal(first[k], bufs2[k]) for k in bufs)
    got, keep = _written(call, kw, bufs)
    untouched = all(bool((bufs[k][keep[k].expand(bufs[k].shape)] == _sentinel(bufs[k].dtype)).all()) for k in keep)
    return got, same, untouched, bufs


def references(call: Call):
    if call.plane is not None:
        return plane_references(call)
    acc = {m: R.tap_sum(call.x.hi, call.x.lo, call.pc, cin_off=call.kw.get("cin_off", 0), frames=call.kw.get("frames"),
                        out_hw=call.kw.get("out_hw"), model=m) for m in (False, True)}
    B, Tt, T, H, W, Ho, Wo = call.kw["geom"]
    kw = dict(call.kw)
    hd = kw["head"]
    if hd is not None:
        kw["head"] = {"w": hd["w"], "b": hd["b"], "sigmoid_mask": hd["sigmoid_mask"]}
    exact, model = R.epilogue(acc[False], call.pc, kw), R.epilogue(acc[True], call.pc, kw)
    scale = {k: max(float(v.abs().max()), 1e-20) for k, v in exact.items()}
    if hd is not None and hd["sigmoid_mask"]:
        # a sigmoid output moves by at most 1/4 of its logit's error: held to a quarter of the logits' max (as the
        # instance-center head is in tests/test_predict_gpu.py), not to the max of the saturated sigmoid
        logits = R.epilogue(acc[False], call.pc, dict(kw, head=dict(kw["head"], sigmoid_mask=0)))
        for k in range(len(hd["outs"])):
            if hd["sigmoid_mask"] >> k & 1:
                scale[f"head{k}"] = max(scale[f"head{k}"], 0.25 * float(logits[f"head{k}"].abs().max()))
    if "col_sums" in exact:       # a column sum is held to the sum of the magnitudes it adds up (it may cancel to ~0)
        scale["col_sums"] = max(float(_activated(acc[False], call).abs().sum(dim=(1, 2)).max()), 1e-20)
    return exact, model, scale


def plane_references(call: Call):
    """(exact = model, {name: summed magnitudes of each element's terms}, scale) of a one-plane call: fp32 output only"""
    geo = dict(cin_off=call.kw.get("cin_off", 0), frames=call.kw.get("frames"), out_hw=call.kw.get("out_hw"))
    acc = R.tap_sum(call.x.hi, None, call.pc, **geo)
    mag = R.tap_sum(call.x.hi, None, call.pc, absolute=True, **geo)
    ib = call.kw.get("img_bias")
    n_img, Ho, Wo, bn = mag.shape
    mag = mag + (ib.double().abs().view(n_img, 1, 1, bn) if ib is not None else call.pc.bias.double().abs().to(DEV))
    mag = mag[..., :call.kw["n_valid"]]
    mags = {"f32": mag if call.kw.get("out_f32_nhwc") else mag.permute(0, 3, 1, 2)}
    exact = R.epilogue(acc, call.pc, call.kw)
    scale = {k: max(float(v.abs().max()), 1e-20) for k, v in exact.items()}
    return exact, mags, scale


def _activated(acc, call):
    kw = {k: v for k, v in call.kw.items() if k != "head"}
    kw["out"], kw["out2"], kw["out_f32"], kw["col_sums"] = True, None, None, None
    kw["n_store"] = call.pc.bn
    return R.epilogue(acc, call.pc, kw)["y"]


def _excess(got, ref, split):
    """max over elements of |got - ref| beyond split * |ref| (0 if every element is inside its split allowance)"""
    return float(((got - ref).abs() - split * ref.abs()).clamp_min(0.0).max())


# ------------------------------------------------------------------------------------------------ coverage
def _groups(taps, stride, mode):
    """Largest run of taps that share one activation load (include/stp3_b200.h, tune_group): consecutive taps with the
    same (dt, dx) whose dy advance by the stride, at most 4; mode 1 never shares."""
    if mode == 1:
        return 1
    gmax, i = 1, 0
    while i < len(taps):
        g = 1
        while (g < 4 and i + g < len(taps) and taps[i + g][0] == taps[i][0] and taps[i + g][2] == taps[i][2] and
               taps[i + g][1] == taps[i][1] + g * stride):
            g += 1
        gmax, i = max(gmax, g), i + g
    return gmax


def tiling(call: Call, cfg):
    """what the library runs for this call and tiling (tests/conv_reference.py tiling)"""
    kw = call.kw
    return R.tiling(call.pc, kw["geom"], cfg, in_cstride=call.x.hi.shape[-1], cin_off=kw.get("cin_off", 0),
                    t0=kw["frames"][0] if kw.get("frames") is not None else 0,
                    n_store=kw.get("n_store", 0) if kw["out"] is not None else 0,
                    one_block=kw["head"] is not None or kw["out2"] is not None, w_img_stride=kw.get("w_img_stride", 0),
                    operand=dense.PLANE_OPERAND[call.plane] if call.plane is not None else 0,
                    n_sm=torch.cuda.get_device_properties(DEV).multi_processor_count)


def instantiation(call: Call, t: dict):
    """conv_igemm_kernel<BN, STACK, FULLK, OP> the call runs: (BN, STACK, FULLK) for hi/lo operands, (plane type, BN,
    FULLK) for one plane"""
    if call.plane is not None:
        return (PLANE_NAMES[call.plane], t["bn_blk"], t["fullk"])
    return (t["bn_blk"], bool(t["stacked"]), t["fullk"])


def features(call: Call, cfg, t: Optional[dict] = None):
    pc, kw = call.pc, call.kw
    t = t if t is not None else tiling(call, cfg)
    B, Tt, T, H, W, Ho, Wo = kw["geom"]
    f = {f"width {pc.bn}" if pc.bn < 256 else "width 256 (two launches)"}
    if t["stacked"]:
        f.add("STACK")
    if t["fullk"]:
        f.add("FULLK")
    f.add("weights resident" if t["resident"] else "weights streamed")
    if pc.k_hi > 0 and pc.k_lo > 0:
        f.add("ks_first > 0")
    if t["bn_blk"] == pc.bn and (pc.cout + 15) // 16 * 16 < pc.bn:
        f.add("n_mma < bn")
    if cfg[1] & 4:
        f.add("streamed (+4)")
    if _groups(pc.taps, pc.stride, cfg[1] & 3) > 1:
        f.add("tap group > 1")
    if pc.stride == 2:
        f.add("stride 2")
    t0 = kw["frames"][0] if kw.get("frames") is not None else 0
    if t0 == 0 and any(dt < 0 for dt, _, _ in pc.taps):
        f.add("causal taps at frame 0")
    if T < Tt:
        f.add("frame window")
    if kw.get("out_hw") is not None:
        f.add("out_hw override")
    if kw.get("cin_off", 0) > 0:
        f.add("cin_off > 0")
    if len(pc.taps) > 27:
        f.add("taps > 27")
    if Tt == 7:
        f.add("T_total 7")
    if call.chunk is not None:
        fn, j, n = call.chunk
        if fn == "conv1x1_raw" and n > 1 and j == n - 1:
            f.add("trunk: last chunk of a forward over 256 columns")
        if fn == "conv1x1_dgrad" and n > 1:
            f.add("trunk: input-gradient chunk of over 256 input channels")
        if call.x.c % 64 or pc.cout % 64:
            f.add("trunk: channels not a multiple of 64")
    f.add(f"res_mode {0 if kw['residual'] is None else 2 if kw.get('res_after_act') else 1}")
    for k, coff in (("out", "out_coff"), ("out2", "out2_coff")):
        if kw[k] is not None:
            f.add("vector store" if kw[k][-1] % 16 == 0 and kw.get(coff, 0) % 16 == 0 else "scalar store")
    if kw["residual"] is not None:
        r = kw["residual"]
        f.add("vector residual" if r.hi.shape[-1] % 16 == 0 and kw.get("res_coff", 0) % 16 == 0 else "scalar residual")
    if kw["out"] is not None:
        f.add("hi/lo output")
        if 0 < kw.get("n_store", 0) < pc.bn:
            f.add("partial n_store")
    if kw["out_f32"] is not None:
        if kw.get("out_f32_nhwc"):
            f.add("f32 NHWC output")
        elif kw.get("sigmoid"):
            f.add("f32 NCHW output + sigmoid")
        else:
            f.add("f32 NCHW output")
    for k, name in (("head", "fused head"), ("out2", "out2"), ("col_sums", "col_sums"), ("img_bias", "img_bias")):
        if kw[k] is not None:
            f.add(name)
    return f


REQUIRED = ["width 64", "width 128", "width 256 (two launches)", "STACK", "FULLK", "ks_first > 0", "n_mma < bn",
            "streamed (+4)", "tap group > 1", "stride 2", "causal taps at frame 0", "frame window", "out_hw override",
            "res_mode 0", "res_mode 1", "res_mode 2", "vector store", "scalar store", "vector residual",
            "scalar residual", "hi/lo output", "f32 NCHW output + sigmoid", "f32 NHWC output", "fused head", "out2",
            "col_sums", "img_bias", "partial n_store", "cin_off > 0", "taps > 27", "T_total 7",
            "trunk: last chunk of a forward over 256 columns", "trunk: input-gradient chunk of over 256 input channels",
            "trunk: channels not a multiple of 64"]


# ------------------------------------------------------------------------------------------------ driver
_RUNS = {}


def run_source(name):
    """Record the source's calls, replay each under (0, 0) and every tuning candidate; cached per module."""
    if name in _RUNS:
        return _RUNS[name]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    calls = SOURCES[name]()
    assert calls, f"{name}: no convolution recorded"
    rows = []
    for i, call in enumerate(calls):
        exact, model, scale = references(call)
        plane = call.plane is not None
        outs = {}
        for cfg in [(0, 0)] + (dense.tune_candidates(call.pc) if call.all_tilings else []):
            got, same, untouched, bufs = _replay(call, cfg)
            assert set(got) == set(exact), (set(got), set(exact))
            e_x = max(float((got[k] - exact[k].reshape(got[k].shape)).abs().max()) / scale[k] for k in got)
            t = tiling(call, cfg)
            K = len(call.pc.taps) * call.pc.cin_p
            row = dict(call=i, source=call.source, cfg=cfg, exact=e_x, same=same, untouched=untouched, plane=plane, K=K, bar=model_bar(K),
                       inst=instantiation(call, t), features=features(call, cfg, t),
                       desc=f"{call.tag + ': ' if call.tag else ''}{len(call.pc.taps)}tap s{call.pc.stride} cin{call.pc.cin_p} "
                            f"bn{call.pc.bn} {call.kw['geom']}" + (f" {PLANE_NAMES[call.plane]}" if plane else ""))
            if plane:       # exact = model; `model` holds the summed magnitudes
                row["model"] = e_x
                row["ulps"] = max(float(((got[k] - exact[k].reshape(got[k].shape)).abs() /
                                         (ULP * model[k].reshape(got[k].shape) + 1e-300)).max()) for k in got)
                outs[cfg[1]] = bufs["out_f32"]
            else:
                row["model"] = max(_excess(got[k], model[k].reshape(got[k].shape), SPLIT if k in ("y", "y2") else 0.0)
                                   / scale[k] for k in got)
            rows.append(row)
        if plane:
            # the stacked operand does not apply to a plane: +8 runs the tiling without it
            for r in rows[-len(outs):]:
                g = r["cfg"][1]
                r["stack_ignored"] = not g & 8 or g & ~8 not in outs or torch.equal(outs[g], outs[g & ~8])
            if call.prod is not None:
                cfg, prod = call.prod
                bufs = _replay(call, cfg)[3]
                for r in rows[-len(outs):]:
                    r["production"] = torch.equal(bufs["out_f32"], prod)
        del exact, model, outs
    del calls
    torch.cuda.empty_cache()
    print(f"\n{name}: {len(rows)} replays in {time.time() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated")
    _RUNS[name] = rows
    return rows


def test_no_call_bypasses_the_recorder():
    assert not bare_conv_calls()


@pytest.mark.parametrize("name", list(SOURCES))
def test_recorded_convolutions_under_every_tiling(name):
    rows = run_source(name)
    worst = {}
    for r in rows:
        w = worst.setdefault(r["call"], dict(desc=r["desc"], exact=0.0, model=0.0, n=0, bar=r["bar"]))
        w["exact"], w["model"], w["n"] = max(w["exact"], r["exact"]), max(w["model"], r["model"]), w["n"] + 1
    print(f"\n{name}: {len(worst)} convolutions, {len(rows)} replays")
    for i, w in sorted(worst.items()):
        print(f"  #{i:<3d} {w['desc']:<60s} tilings {w['n']}  exact {w['exact']:.2e}  model {w['model']:.2e} "
              f"(bar {w['bar']:.1e})")
    if any(r["plane"] for r in rows):
        print(f"  one-plane: worst {max(r['ulps'] for r in rows):.1f} fp32 ulps of the summed magnitudes "
              f"(bar {CONV_ULPS})")
    bad = [(r["call"], r["cfg"], r["exact"], r["model"], r["same"], r["untouched"]) for r in rows if not passed(r)]
    assert not bad, bad


def passed(r):
    if r["plane"]:          # exact = model: the model bar and the ulp bar
        return (r["model"] <= r["bar"] and r["ulps"] <= CONV_ULPS and r["same"] and r["untouched"] and
                r["stack_ignored"] and r.get("production", True))
    return r["exact"] <= EXACT_BAR and r["model"] <= r["bar"] and r["same"] and r["untouched"]


REQUIRED_PLANE = ["n_mma < bn", "stride 2", "out_hw override", "causal taps at frame 0", "img_bias", "f32 NHWC output",
                  "f32 NCHW output + sigmoid", "frame window", "ks_first > 0", "width 256 (two launches)"]


def _worst_by_k(rows):
    """{(plane type, K): (worst model error of max |model|, worst ulps)} over one-plane replays"""
    worst = {}
    for r in rows:
        if r["plane"]:
            key = (r["inst"][0], r["K"])
            w = worst.get(key, (0.0, 0.0))
            worst[key] = (max(w[0], r["model"]), max(w[1], r["ulps"]))
    return worst


def test_every_instantiation_and_feature_is_replayed():
    rows = [r for name in SOURCES for r in run_source(name)]
    insts = {}
    for r in rows:
        d = insts.setdefault(r["inst"], {"replays": 0, "group": 0, "+4": 0, "streamed": 0, "resident": 0})
        d["replays"] += 1
        d["+4"] += "streamed (+4)" in r["features"]
        d["group"] += "tap group > 1" in r["features"]
        d["streamed"] += "weights streamed" in r["features"]
        d["resident"] += "weights resident" in r["features"]
    hilo, plane = [r for r in rows if not r["plane"]], [r for r in rows if r["plane"]]
    counts = {f: sum(f in r["features"] for r in hilo) for f in REQUIRED}
    counts_plane = {f: sum(f in r["features"] for r in plane) for f in REQUIRED_PLANE}
    print("\ninstantiation (BN, STACK, FULLK) / (plane, BN, FULLK): replays / with a tap group > 1 / under a +4 tiling / "
          "weights streamed / weights resident")
    for k in sorted(insts, key=str):
        d = insts[k]
        print(f"  {k}: {d['replays']} / {d['group']} / {d['+4']} / {d['streamed']} / {d['resident']}")
    print("feature: hi/lo replays")
    for f in REQUIRED:
        print(f"  {f:<28s} {counts[f]}")
    print("feature: one-plane replays")
    for f in REQUIRED_PLANE:
        print(f"  {f:<28s} {counts_plane[f]}")
    print("one-plane worst per K: model error of max |model| / fp32 ulps of the summed magnitudes")
    for (m, K), (e, u) in sorted(_worst_by_k(rows).items()):
        print(f"  {m} K {K:<6d} {e:.2e} (bar {model_bar(K):.1e})  {u:5.1f} ulps")
    expected = {(bn, st, fk) for bn in (64, 128) for st in (False, True) for fk in (False, True) if not (st and bn == 128)}
    expected |= {(m, bn, fk) for m in PLANE_NAMES.values() for bn in (64, 128) for fk in (False, True)}
    assert set(insts) == expected, set(insts) ^ expected
    assert all(d["group"] and d["+4"] and d["streamed"] for d in insts.values()), insts
    assert all(d["resident"] for k, d in insts.items() if isinstance(k[0], str)), insts
    assert all(counts.values()), [f for f, c in counts.items() if not c]
    assert all(counts_plane.values()), [f for f, c in counts_plane.items() if not c]
    recorded = [r for r in plane if not r["source"].startswith("synthetic")]
    assert recorded and all("production" in r for r in recorded)
