"""GPU: the eval-mode planner (stp3_plan_maps / stp3_plan_cost / stp3_plan_refine behind Cost_Function and Planning)
against the fp64 oracle (oracle/torch_planning.py, itself pinned to the unmodified reference by
tests/test_planning_cpu.py): index-exact footprint and cell sampling, the general costs, the selection within each
command window, both progress branches, a whole Planning-configuration STP3 as evaluate.py calls it, no host
synchronisation, and determinism."""
import copy

import numpy as np
import pytest
import torch

from oracle import lift_splat_oracle as O
from oracle import torch_dense as TD
from oracle import torch_planning as TP
from oracle import torch_predict as TPR
from oracle.make_golden_planning import CASES, case_inputs, footprints, planning_cfg, planning_module
from stp3_b200 import dense
from stp3_b200.cost import Cost_Function
from stp3_b200.utils import geometry as G
from stp3_b200.utils import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FACTOR = {"safety": "safetycost", "headway": "headwaycost", "lrdivider": "lrdividercost", "costvolume": "costvolume",
          "rule": "rulecost", "comfort": "comfortcost", "progress": "progresscost"}


def on_gpu(x):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in x.items()}


def rel_to_max(got, ref):
    ref = ref.double().cpu()
    return (got.double().cpu() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


# ------------------------------------------------------------------------------------------------ exact indices
def special_values(dx, bx, lo, hi, gen, n):
    """Coordinates on cell boundaries of both index expressions (k * dx for get_points, bx + k * dx for discretize),
    1 ulp either side of them, negative ones and positions off the grid, as fp32."""
    k = torch.arange(lo, hi, dtype=torch.float32)
    base = torch.cat([k * dx, bx + k * dx, torch.tensor([-80.0, -60.5, 60.5, 80.0, -0.0, 0.0])])
    v = torch.cat([base, torch.nextafter(base, torch.tensor(float("inf"))),
                   torch.nextafter(base, torch.tensor(float("-inf")))])
    return v[torch.randint(0, v.numel(), (n,), generator=gen)]


def exact_inputs(carla, B=2, seed=0):
    cfg = planning_cfg(carla)
    N, T = cfg.PLANNING.SAMPLE_NUM, cfg.N_FUTURE_FRAMES
    X = 200
    dx = float(torch.tensor(cfg.LIFT.X_BOUND[2], dtype=torch.float32))
    bx = float(torch.tensor(cfg.LIFT.X_BOUND[0] + cfg.LIFT.X_BOUND[2] / 2.0, dtype=torch.float32))
    g = torch.Generator().manual_seed(seed)
    n = B * N * T
    lim = int(cfg.LIFT.X_BOUND[1] / cfg.LIFT.X_BOUND[2]) + 30
    trajs = torch.stack([special_values(dx, bx, -lim, lim, g, n), special_values(dx, bx, -lim, lim, g, n),
                         torch.zeros(n)], -1).view(B, N, T, 3)
    hd = torch.stack([(torch.randint(0, 12, (B, X, X), generator=g) == 0).float(),
                      (torch.randint(0, 3, (B, X, X), generator=g) != 0).float()], 1)
    return dict(trajs=trajs, cost_volume=syn.exact_gauss((B, T, X, X), g) * 32.0,
                semantic_pred=torch.randint(0, 8, (B, T, X, X), generator=g) == 0, hd_map=hd,
                target_points=torch.randint(-256, 257, (B, 2), generator=g).float() / 16.0)


def one_term_cost_function(carla, term, w=(1.0, 1.0), factor=1.0):
    cf = Cost_Function(planning_cfg(carla))
    for t, child in FACTOR.items():
        getattr(cf, child).factor = factor if t == term else 0.0
    cf.safetycost.w.data = torch.tensor(w)
    return cf


@pytest.mark.parametrize("carla", [False, True], ids=["nuscenes", "carla"])
@pytest.mark.parametrize("term, w, factor", [("safety", (1.0, 0.0), 1.0), ("safety", (0.0, 1.0), 2.0 ** -12),
                                             ("headway", None, 1.0), ("lrdivider", None, 1.0),
                                             ("costvolume", None, 1.0), ("rule", None, 0.25)])
def test_footprint_and_cell_indices_are_exact(carla, term, w, factor):
    """One term at a time on binary maps, with factors that keep the counts below the clamp at 100: the count terms
    (and the gathered cost volume) equal the oracle exactly, so
    every footprint cell and discretised cell is the reference's.  The lane cost and the velocity-weighted count carry
    an fp32 square root: they are held to 1e-6 of each entry (of the lane cost's max), far below the step a wrong index
    makes."""
    cf = one_term_cost_function(carla, term, w or (1.0, 1.0), factor)
    x = exact_inputs(carla)
    lane, drv = x["hd_map"][:, 0:1], x["hd_map"][:, 1:2]
    fps = (cf._pack()["fp0"], cf._pack()["fp1"])
    ref = TP.terms(cf, x["cost_volume"], x["trajs"], x["semantic_pred"], lane, drv, x["target_points"], fps)[term]
    cf = cf.to(DEV)
    xg = on_gpu(x)
    fc, fo = cf(xg["cost_volume"], xg["trajs"], xg["semantic_pred"], lane.to(DEV), drv.to(DEV), xg["target_points"])
    assert fc.abs().max().item() == 0.0
    got = fo.double().cpu()
    assert ref.abs().max() > 0, "the case exercises nothing"
    if term == "lrdivider":        # (L - d)^2 near d = L magnifies the square root's rounding: 1e-6 of max
        bad = (got - ref).abs() > 1e-6 * ref.abs().max()
    elif term == "safety" and w[1] != 0:
        bad = (got - ref).abs() > 1e-6 * ref.abs()
    else:
        bad = got != ref
    assert not bad.any(), (term, int(bad.sum()), got[bad][:5], ref[bad][:5])


# ------------------------------------------------------------------------------------------------ general costs
def assert_logits_off_ties(hd):
    if hd.shape[1] == 4:
        for c in (0, 2):
            p = torch.softmax(hd[:, c:c + 2].double(), 1)[:, 1]
            assert (p - 0.5).abs().min().item() >= 1e-5


@pytest.mark.parametrize("case", list(CASES))
def test_costs_match_fp64(case):
    m = planning_module(CASES[case]["carla"])
    x = case_inputs(case)
    assert_logits_off_ties(x["hd_map"])
    lane, drv = m.split_hd_map(x["hd_map"])
    fc64, fo64 = TP.cost_function(m.cost_function, x["cost_volume"], x["trajs"], x["semantic_pred"], lane, drv,
                                  x["target_points"], footprints(m))
    m = m.to(DEV)
    xg = on_gpu(x)
    lane, drv = m.split_hd_map(xg["hd_map"])
    fc, fo = m.cost_function(xg["cost_volume"], xg["trajs"], xg["semantic_pred"], lane, drv, xg["target_points"])
    torch.cuda.synchronize()
    assert rel_to_max(fc, fc64) < 1e-5, rel_to_max(fc, fc64)
    assert rel_to_max(fo, fo64) < 1e-5, rel_to_max(fo, fo64)
    print(f"{case}: cost_fc {rel_to_max(fc, fc64):.2e}, cost_fo {rel_to_max(fo, fo64):.2e} of max")


@pytest.mark.parametrize("targets, uses_target", [([[0.0, 0.0], [0.0, 0.0]], False), ([[0.3, -0.2], [0.1, 0.2]], False),
                                                  ([[0.3, -0.2], [0.1, 0.3]], True), ([[-4.0, 10.0], [2.5, 7.0]], True)])
def test_progress_branch(targets, uses_target):
    """Progress drops its target term when target_points.sum() < 0.5 over the whole batch, including non-zero
    targets whose sum is below 0.5."""
    cf = one_term_cost_function(False, "progress")
    x = case_inputs("nuscenes_hd2")
    tp = torch.tensor(targets)
    assert (tp.sum().item() >= 0.5) == uses_target
    lane, drv = x["hd_map"][:, 0:1], x["hd_map"][:, 1:2]
    t = TP.terms(cf, x["cost_volume"], x["trajs"], x["semantic_pred"], lane, drv, tp, (cf._pack()["fp0"],
                                                                                       cf._pack()["fp1"]))
    cf = cf.to(DEV)
    fc, fo = cf(x["cost_volume"].to(DEV), x["trajs"].to(DEV), x["semantic_pred"].to(DEV), lane.to(DEV), drv.to(DEV),
                tp.to(DEV))
    assert fo.abs().max().item() == 0.0
    assert rel_to_max(fc, t["progress"]) < 1e-5
    no_target = -x["trajs"][..., 1].double().max(-1).values * cf.progresscost.factor
    assert torch.equal(t["progress"], torch.clamp(no_target, -100, 100)) != uses_target


# ------------------------------------------------------------------------------------------------ selection
def run_planning(m, x):
    """Planning.forward's stages, returning the selected index as well; checks forward() gives the same trajectory."""
    lane, drv = m.split_hd_map(x["hd_map"])
    B, N = x["trajs"].shape[:2]
    win = m.windows(x["commands"], B, N, DEV)
    h0 = m.reduce(x["cam_front"])
    fc, fo = m.cost_function(x["cost_volume"], x["trajs"], x["semantic_pred"], lane, drv, x["target_points"])
    out, sel = m._refine(h0, x["trajs"], win, fc, fo, x["target_points"], lane.shape[1])
    _, out2 = m(x["cam_front"], x["trajs"], None, x["cost_volume"], x["semantic_pred"], x["hd_map"], x["commands"],
                x["target_points"])
    assert torch.equal(out, out2)
    return out, sel


def check_selection(m64, fps, x, out, sel, tag):
    fc, fo = TP.cost_function(m64.cost_function, x["cost_volume"], x["trajs"], x["semantic_pred"],
                              *m64.split_hd_map(x["hd_map"].cpu()), x["target_points"], fps)
    cs = fc + fo.sum(-1)
    sel = sel.cpu().long()
    for b, (s, c) in enumerate(TP.windows(x["commands"], x["trajs"].shape[1])):
        assert s <= sel[b] < s + c, (tag, b, int(sel[b]), s, c)
        best = cs[b, s:s + c].min()
        assert cs[b, sel[b]] - best <= 1e-5 * cs.abs().max(), (tag, b, float(cs[b, sel[b]]), float(best))
    ref, _, _, _ = TP.planning_forward(m64, fps, **{k: (v.cpu() if torch.is_tensor(v) else v) for k, v in x.items()},
                                       selected=sel)
    e = rel_to_max(out, ref)
    assert e < 2e-4, (tag, e)
    assert torch.all(out[..., 2] == 0)
    print(f"{tag}: selected {sel.tolist()}, output_traj {e:.2e} of max")


@pytest.mark.parametrize("case", list(CASES))
def test_selection_and_refinement(case):
    m = planning_module(CASES[case]["carla"])
    fps = footprints(m)
    m64 = copy.deepcopy(m)
    x = case_inputs(case)
    out, sel = run_planning(m.to(DEV), on_gpu(x))
    check_selection(m64, fps, x, out, sel, case)


def test_ties_pick_the_lowest_index():
    """Exact duplicates score equal (the reference stacks the chosen third three times): the lowest index wins."""
    m = planning_module(False)
    x = case_inputs("nuscenes")
    k = 600
    for b, (s, c) in enumerate(TP.windows(x["commands"], 1800)):
        x["trajs"][b, s:s + c] = x["trajs"][b, s + 7].clone()
    out, sel = run_planning(m.to(DEV), on_gpu(x))
    assert sel.tolist() == [0, k, 2 * k, 0]


# ------------------------------------------------------------------------------------------------ whole model
def small_planning_model():
    """A Planning-configuration STP3 on a 32 x 32 BEV with 96 x 96 images: cam_front is 64 x 12 x 12, reduced to
    8 x 2 x 2 = 32 values, so the GRU state is 32."""
    from oracle.make_golden_predict import build_prediction_model
    from stp3_b200.config import PLANNING_OVERRIDES, get_cfg
    cfg = get_cfg(PLANNING_OVERRIDES, perception=False).merge({
        "LIFT": {"X_BOUND": [-8.0, 8.0, 0.5], "Y_BOUND": [-8.0, 8.0, 0.5], "D_BOUND": [2.0, 10.0, 1.0]},
        "IMAGE": {"FINAL_DIM": (96, 96)}, "PLANNING": {"GRU_STATE_SIZE": 32, "SAMPLE_NUM": 300}})
    model = build_prediction_model(cfg)
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(96, 96), out_channels=64, n_cameras=2, receptive_field=3)
    return model, lcfg


def test_planning_config_end_to_end(monkeypatch):
    model, lcfg = small_planning_model()
    # build_prediction_model's init_exact randomised the cost function's geometry: put it back
    model.planning.cost_function.load_state_dict(Cost_Function(model.cfg).state_dict())
    m64 = copy.deepcopy(model).double()
    fps = footprints(model.planning)
    inp = syn.lift_inputs(lcfg, 1, seed=5, random_pose=True)
    model = model.to(DEV)
    rec = {}
    predict_hl = model._predict_hl

    def record(states):                 # the future frames the decoder receives
        y = predict_hl(states)
        rec["frames"] = dense.to_f32(y, 0, 64)
        return y
    monkeypatch.setattr(model, "_predict_hl", record)
    with torch.no_grad():
        out = model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                     inp["extrinsics"], inp["future_egomotion"])
    torch.cuda.synchronize()
    assert torch.equal(out["cam_front"].cpu(), inp["feat"][:, -1, 1])
    # the costvolume head against the fp64 model oracle, on the frames the GPU's prediction stage produced (the
    # recurrent stage amplifies its inputs' rounding, so the chained fp64 model is reported, not held to a bar)
    dec = TD.decoder(rec["frames"].double().cpu(), m64.decoder)["costvolume"]
    e = rel_to_max(out["costvolume"], dec)
    assert e < 3e-4, e
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(lcfg.final_dim, lcfg.downsample, lcfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(lcfg.x_bound, lcfg.y_bound, lcfg.z_bound)
    ora = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), cam_M.numpy(), cam_t.numpy(), ego_R.numpy(),
                       ego_t.numpy(), xs.numpy(), ys.numpy(), ds.numpy(), G.bev_offset(start, res).numpy(),
                       res.numpy(), dim.numpy(), lcfg.discount)
    with torch.no_grad():
        bev = torch.from_numpy(ora["bev"])
        ego = inp["future_egomotion"].double()
        ego = torch.cat([torch.zeros_like(ego[:, :1]), ego[:, :-1]], 1)
        X = bev.shape[-1]
        bev = torch.cat([bev, ego.view(1, 3, 6, 1, 1).expand(1, 3, 6, X, X)], dim=2)
        ref = TPR.predict_and_decode(TD.temporal_model(bev, m64.temporal_model), m64)
    print(f"end to end: costvolume {e:.2e} of max vs fp64 on its own frames, "
          f"{rel_to_max(out['costvolume'], ref['costvolume']):.2e} vs the chained fp64 model")
    # model.planning exactly as evaluate.py:121-131 calls it, on what the GPU produced
    n_present = model.receptive_field
    seg = torch.argmax(out["segmentation"], dim=2, keepdim=True)
    ped = torch.argmax(out["pedestrian"], dim=2, keepdim=True)
    occupancy = torch.logical_or(seg, ped)
    g = torch.Generator().manual_seed(9)
    N, T = 300, model.n_future
    trajs = torch.stack([(torch.randint(-32, 33, (1, N, T), generator=g).float() / 32.0).cumsum(-1),
                         (torch.randint(0, 129, (1, N, T), generator=g).float() / 64.0).cumsum(-1),
                         torch.zeros(1, N, T)], -1)
    target = torch.zeros(1, 2)
    x = dict(cam_front=out["cam_front"].detach(), trajs=trajs.to(DEV), cost_volume=out["costvolume"][:, n_present:],
             semantic_pred=occupancy[:, n_present:].squeeze(2), hd_map=out["hdmap"].detach(), commands=["FORWARD"],
             target_points=target.to(DEV))
    with torch.no_grad():
        _, final_traj = model.planning(cam_front=x["cam_front"], trajs=x["trajs"], gt_trajs=None,
                                       cost_volume=x["cost_volume"], semantic_pred=x["semantic_pred"],
                                       hd_map=x["hd_map"], commands=x["commands"], target_points=x["target_points"])
        out2, sel = run_planning(model.planning, x)
    assert final_traj.shape == (1, T, 3) and torch.equal(final_traj, out2)
    check_selection(m64.planning, fps, x, out2, sel, "end to end")


# ------------------------------------------------------------------------------------------------ host sync, determinism
def test_no_host_synchronisation_and_determinism():
    m = planning_module(True).to(DEV)
    x = on_gpu(case_inputs("carla"))
    args = (x["cam_front"], x["trajs"], None, x["cost_volume"], x["semantic_pred"], x["hd_map"], x["commands"],
            x["target_points"])
    with torch.no_grad():
        _, first = m(*args)                 # packs the weights and reads the footprints once
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _, second = m(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(first, second)
    assert np.isfinite(first.cpu().numpy()).all()
