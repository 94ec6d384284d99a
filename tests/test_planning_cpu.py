"""CPU: the eval-mode planner's fp64 oracle against the unmodified reference (tests/golden/planning_*.npz,
oracle/make_golden_planning.py), the ego footprints, checkpoint compatibility of the Planning head, and every refusal of
the modules and of the C ABI's planning entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import torch_planning as TP
from oracle.make_golden_planning import CASES, case_inputs, footprints, planning_module
from stp3_b200 import _lib
from stp3_b200.config import PLANNING_CARLA_OVERRIDES, PLANNING_OVERRIDES, PREDICTION_OVERRIDES, get_cfg
from stp3_b200.cost import footprint, gen_dx_bx
from stp3_b200.layers.convolutions import Bottleneck
from stp3_b200.models.planning_model import Planning
from stp3_b200.models.stp3 import STP3

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(case):
    return np.load(os.path.join(GOLDEN, f"planning_{case}.npz"))


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(case):
    """The fp64 oracle, recomputed here, equals the one stored next to the reference's values, and both agree with the
    reference: costs to fp32 rounding, the same selected candidates, the output trajectory to 1e-5 of max."""
    g = _golden(case)
    m = planning_module(CASES[case]["carla"])
    x = case_inputs(case)
    with torch.no_grad():
        out, sel, fc, fo = TP.planning_forward(m, footprints(m), **x)
    for name, a in (("cost_fc", fc), ("cost_fo", fo)):
        idx, ref, ora, mx = g[f"{name}_idx"], g[f"{name}_ref"], g[f"{name}_ora"], float(g[f"{name}_max"])
        got = a.reshape(-1).numpy()[idx]
        np.testing.assert_allclose(got, ora, rtol=0, atol=1e-12 * mx)
        assert np.abs(ref - ora).max() <= 1e-6 * mx, (name, np.abs(ref - ora).max() / mx)
        assert abs(a.abs().max().item() - mx) <= 1e-12 * mx
    assert sel.tolist() == g["sel_ora"].tolist() == g["sel_ref"].tolist()
    np.testing.assert_allclose(out.numpy(), g["out_ora"], rtol=0, atol=1e-12 * np.abs(g["out_ora"]).max())
    assert np.abs(g["out_ref"] - g["out_ora"]).max() <= 1e-5 * np.abs(g["out_ora"]).max()


@pytest.mark.parametrize("overrides, counts", [(PLANNING_OVERRIDES, (32, 192)), (PLANNING_CARLA_OVERRIDES, (250, 4500))])
def test_footprint_cells(overrides, counts):
    cfg = get_cfg(overrides, perception=False)
    dx, bx = gen_dx_bx(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
    lam = int(cfg.COST_FUNCTION.LAMBDA / dx[0])          # cost.py:110, in fp32
    assert lam == (5 if overrides is PLANNING_CARLA_OVERRIDES else 2)
    for lam_, n in zip((0, lam), counts):
        r0, r1, c0, c1 = footprint(cfg.EGO.WIDTH, cfg.EGO.HEIGHT, dx[:2], bx[:2], lam_)
        assert (r1 - r0 + 1) * (c1 - c0 + 1) == n
        # no edge within 1e-6 of a cell: skimage's boundary rule never decides (footprint() also refuses that)
        d, b = dx[:2].double().numpy(), bx[:2].double().numpy()
        H, W = cfg.EGO.HEIGHT, cfg.EGO.WIDTH
        edges = [(-H / 2 + 0.5 - lam_ - b[0]) / d[0], (H / 2 + 0.5 + lam_ - b[0]) / d[0],
                 (-W / 2 - lam_ - b[1]) / d[1], (W / 2 + lam_ - b[1]) / d[1]]
        assert min(abs(e - round(e)) for e in edges) > 1e-6


def test_footprint_refuses_an_edge_on_a_cell():
    dx, bx = torch.tensor([0.5, 0.5]), torch.tensor([-49.75, -49.75])
    with pytest.raises(ValueError, match="boundary rule"):
        footprint(2.5, 4.0, dx, bx)      # -W/2 = -1.25 -> column 97.0 exactly


@pytest.mark.parametrize("case, overrides", [("nuscenes", PLANNING_OVERRIDES), ("carla", PLANNING_CARLA_OVERRIDES)])
def test_reference_checkpoint_keys_load_strict(case, overrides):
    g = _golden(case)
    sd = {k: torch.zeros([int(v) for v in s.split(",") if v]) for k, s in zip(g["ref_keys"], g["ref_shapes"])}
    model = STP3(get_cfg(overrides, perception=False), backbone=torch.nn.Identity())
    model.planning.load_state_dict(sd, strict=True)
    assert {"planning." + k for k in sd} <= set(model.state_dict())


def test_planning_head_shapes():
    for ov, g in ((PLANNING_OVERRIDES, 256), (PLANNING_CARLA_OVERRIDES, 128)):
        model = STP3(get_cfg(ov, perception=False), backbone=torch.nn.Identity())
        assert model.planning.GRU.hidden_size == g
        assert model.cfg.PLANNING.COMMAND == ['LEFT', 'FORWARD', 'RIGHT']
        assert all(isinstance(v, float) for v in model.cfg.COST_FUNCTION.values())


def test_command_windows():
    m = planning_module(False)
    assert TP.windows(['LEFT', 'FORWARD', 'RIGHT', 'GO'], 1800) == [(0, 600), (600, 600), (1200, 600), (0, 1800)]
    with pytest.raises(ValueError, match="commands"):
        m.windows(['LEFT'], 2, 1800, "cpu")
    with pytest.raises(ValueError, match="SAMPLE_NUM"):
        m.windows(['LEFT'], 1, 900, "cpu")


@pytest.mark.parametrize("over, needle", [
    ({"N_FUTURE_FRAMES": 0}, "N_FUTURE_FRAMES = 0"),
    ({"SEMANTIC_SEG": {"HDMAP": {"ENABLED": False}}}, "PLANNING.ENABLED needs"),
    ({"SEMANTIC_SEG": {"PEDESTRIAN": {"ENABLED": False}}}, "PLANNING.ENABLED needs"),
])
def test_unsupported_planning_configs_are_refused(over, needle):
    cfg = get_cfg(PLANNING_OVERRIDES, perception=False).merge(over)
    with pytest.raises(NotImplementedError, match=needle):
        STP3(cfg, backbone=torch.nn.Identity())


def test_prediction_config_with_planning_is_refused():
    cfg = get_cfg(PREDICTION_OVERRIDES, perception=False).merge({"PLANNING": {"ENABLED": True}})
    with pytest.raises(NotImplementedError, match="PLANNING"):
        STP3(cfg, backbone=torch.nn.Identity())


def test_planning_module_refusals():
    cfg = get_cfg(PLANNING_OVERRIDES, perception=False)
    with pytest.raises(ValueError, match="GRU state has 128"):
        Planning(cfg, 64, 6, gru_state_size=128)       # 8 x 4 x 8 = 256 reduced values
    with pytest.raises(NotImplementedError, match="multiple of 32"):
        Planning(cfg, 64, 6, gru_state_size=250)
    with pytest.raises(NotImplementedError, match="gru_input_size"):
        Planning(cfg, 64, 5)
    m = Planning(cfg, 64, 6)
    with pytest.raises(NotImplementedError, match="eval-only"):
        m.train()(None, None, None, None, None, None, None, None)
    with pytest.raises(NotImplementedError, match="channels"):
        Planning.split_hd_map(torch.zeros(1, 3, 4, 4))
    with pytest.raises(NotImplementedError, match="k = 1"):
        m.eval().select(None, None, None, None, None, None, k=3)
    non_square = get_cfg(PLANNING_OVERRIDES, perception=False).merge({"LIFT": {"Y_BOUND": [-50.0, 50.0, 1.0]}})
    with pytest.raises(NotImplementedError, match="square"):
        Planning(non_square, 64, 6)


def test_bottleneck_forms():
    b = Bottleneck(32, 8)
    assert b.layers.conv.stride == (1, 1) and not hasattr(b.projection, "upsample_skip_proj")
    assert set(b.projection.state_dict()) == {"conv_skip_proj.weight", "bn_skip_proj.weight", "bn_skip_proj.bias",
                                              "bn_skip_proj.running_mean", "bn_skip_proj.running_var",
                                              "bn_skip_proj.num_batches_tracked"}
    assert Bottleneck(64, 32, downsample=True).layers.conv.stride == (2, 2)
    for kw in ({"in_channels": 32, "out_channels": 32}, {"in_channels": 32, "upsample": True},
               {"in_channels": 32, "out_channels": 8, "kernel_size": 5}, {"in_channels": 32, "out_channels": 8, "dilation": 2}):
        with pytest.raises(NotImplementedError, match="Bottleneck"):
            Bottleneck(**kw)


# ------------------------------------------------------------------------------------------------ C ABI
FAKE = 1 << 20


def plan_desc(**kw):
    f = dict(B=2, N=1800, T=6, H=200, W=200, dx=(0.5, 0.5), bx=(-49.75, -49.75), fp0=(97, 104, 98, 101),
             fp1=(93, 108, 94, 105), safety=1.0, headway=1.0, lrdivider=10.0, comfort=0.1, progress=0.5, volume=100.0,
             rule=5.0, safety_w=(1.0, 1.0), headway_dist=10.0, lane_dist=1.0, n_hd=2, traj_c=3, G=256)
    f.update(kw)
    for k in ("dx", "bx", "safety_w"):
        f[k] = (ctypes.c_float * 2)(*f[k])
    for k in ("fp0", "fp1"):
        f[k] = (ctypes.c_int * 4)(*f[k])
    return _lib.PlanDesc(**f)


def _maps(d, null=False):
    return _lib.lib().stp3_plan_maps(d, None if null else FAKE, FAKE, FAKE, FAKE, FAKE, None)


def _cost(d, null=False):
    return _lib.lib().stp3_plan_cost(d, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None if null else FAKE, None)


def _refine(d, windows=((0, 600), (600, 1200)), null=False):
    flat = [v for w in windows for v in w]
    host = (ctypes.c_int * max(len(flat), 1))(*flat)
    args = [FAKE] * 16
    if null:
        args[3] = None
    return _lib.lib().stp3_plan_refine(d, ctypes.cast(host, ctypes.c_void_p), *args, None)


def test_plan_descriptor_rules():
    """One descriptor per rule, each refused with STP3_EINVAL (-1) and its own message before anything is
    dereferenced; each rule reads a different field, which also pins the ctypes mirror's layout."""
    L = _lib.lib()
    cases = {
        "B, N and T must be positive": lambda: _maps(plan_desc(B=0)),
        "N and T must be positive": lambda: _cost(plan_desc(N=-3)),
        "T must be positive": lambda: _refine(plan_desc(T=0)),
        "T = 17 future frames, at most 16": lambda: _cost(plan_desc(T=17)),
        "N = 1801 is not divisible by 3": lambda: _maps(plan_desc(N=1801)),
        "non-square grid 200 x 100": lambda: _cost(plan_desc(W=100)),
        "dx must be positive": lambda: _maps(plan_desc(dx=(0.0, 0.5))),
        "spans more than 8 cells": lambda: _maps(plan_desc(lane_dist=5.0)),
        "n_hd = 3": lambda: _cost(plan_desc(n_hd=3)),
        "traj_c = 4": lambda: _cost(plan_desc(traj_c=4)),
        "footprint fp0": lambda: _cost(plan_desc(fp0=(104, 97, 98, 101))),
        "footprint fp1": lambda: _maps(plan_desc(fp1=(-1, 108, 94, 105))),
        "larger than 65536 cells": lambda: _cost(plan_desc(fp1=(0, 300, 0, 300))),
        "G = 250 must be a multiple of 32": lambda: _refine(plan_desc(G=250)),
        "G = 1024 must be a multiple of 32": lambda: _refine(plan_desc(G=1024)),
        "G = 0 must be": lambda: _refine(plan_desc(G=0)),
        "window (1200, 601) of sample 1 is outside [0, 1800)": lambda: _refine(plan_desc(),
                                                                               windows=((0, 600), (1200, 601))),
        "window (-1, 600) of sample 0": lambda: _refine(plan_desc(), windows=((-1, 600), (0, 600))),
        "window (0, 0) of sample 0": lambda: _refine(plan_desc(), windows=((0, 0), (0, 600))),
        "stp3_plan_maps: null pointer": lambda: _maps(plan_desc(), null=True),
        "stp3_plan_cost: null pointer": lambda: _cost(plan_desc(), null=True),
        "stp3_plan_refine: null pointer": lambda: _refine(plan_desc(), null=True),
        "desc is null": lambda: L.stp3_plan_maps(None, FAKE, FAKE, FAKE, FAKE, FAKE, None),
    }
    for msg, call in cases.items():
        assert call() == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())


def test_plan_ops_refuse_cpu_tensors():
    from stp3_b200 import ops
    t = torch.zeros(1, 3, 1, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.plan_cost(plan_desc(B=1, N=3, T=1), t, t, t, t, t, t)
