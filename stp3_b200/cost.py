"""The planner's cost function (stp3/cost.py) with the reference's module tree, parameter names and call surface, eval
on sm_90a.  The seven cost terms are children that carry the reference's parameters (dx, bx, and SafetyCost.w) and
constants, so a checkpoint's `planning.cost_function.*` keys load with strict=True; Cost_Function.forward evaluates all
seven at once with two launches (stp3_plan_maps, stp3_plan_cost; DESIGN.md §3.17).

The ego footprint replaces skimage.draw.polygon: footprint() rasterises the rectangle BaseCost.get_origin_points builds
(cost.py:68-81) into the integer (row, col) cells strictly inside it, rows and columns clipped at 0 as skimage does.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .layers._packing import PackedModule
from .utils import geometry as G


def gen_dx_bx(xbound, ybound, zbound):
    """stp3/utils/tools.py:176-181: fp32 cell size and first-cell centre per axis."""
    dx = torch.tensor([row[2] for row in (xbound, ybound, zbound)], dtype=torch.float32)
    bx = torch.tensor([row[0] + row[2] / 2.0 for row in (xbound, ybound, zbound)], dtype=torch.float32)
    return dx, bx


def footprint(width: float, height: float, dx, bx, lambda_=0.0, tol: float = 1e-6):
    """(first row, last row, first column, last column) of the cells strictly inside the ego rectangle of
    get_origin_points(lambda_): vertices in float64 from the fp32 dx / bx, rows from the longitudinal extent, columns from
    the lateral one, both clipped at 0.  An edge within `tol` of a cell centre would leave the choice to skimage's
    boundary rule, which this rasteriser does not reproduce: such a footprint is refused."""
    dx = np.asarray(dx, dtype=np.float32)[:2]
    bx = np.asarray(bx, dtype=np.float32)[:2]
    lo = (np.array([-height / 2. + 0.5 - lambda_, -width / 2. - lambda_]) - bx) / dx
    hi = (np.array([height / 2. + 0.5 + lambda_, width / 2. + lambda_]) - bx) / dx
    for v in (*lo, *hi):
        if abs(v - round(v)) < tol:
            raise ValueError(f"footprint edge {v!r} lies on a cell: skimage's boundary rule would decide it")
    r0, c0 = (max(math.floor(v) + 1, 0) for v in lo)
    r1, c1 = (math.floor(v) for v in hi)
    return int(r0), int(r1), int(c0), int(c1)


class BaseCost(nn.Module):
    """dx / bx (fp32 parameters, as the reference keeps them), the BEV dimension and the ego size.  The terms are
    evaluated together by Cost_Function: calling one on its own is not supported."""

    def __init__(self, cfg):
        super().__init__()
        dx, bx = gen_dx_bx(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        self.dx = nn.Parameter(dx[:2], requires_grad=False)
        self.bx = nn.Parameter(bx[:2], requires_grad=False)
        _, _, self.bev_dimension = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND,
                                                                         cfg.LIFT.Z_BOUND)
        self.W = cfg.EGO.WIDTH
        self.H = cfg.EGO.HEIGHT


class Cost_Volume(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.factor = cfg.COST_FUNCTION.VOLUME


class Rule(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.factor = 5


class SafetyCost(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.w = nn.Parameter(torch.tensor([1., 1.]), requires_grad=False)
        self._lambda = cfg.COST_FUNCTION.LAMBDA
        self.factor = cfg.COST_FUNCTION.SAFETY


class HeadwayCost(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.L = 10     # metres kept to the vehicle ahead
        self.factor = cfg.COST_FUNCTION.HEADWAY


class LR_divider(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.L = 1      # metres kept to the lane divider
        self.factor = cfg.COST_FUNCTION.LRDIVIDER


class Comfort(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.c_lat_acc = 3
        self.c_lon_acc = 3
        self.c_jerk = 1
        self.factor = cfg.COST_FUNCTION.COMFORT


class Progress(BaseCost):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.factor = cfg.COST_FUNCTION.PROGRESS


class Cost_Function(PackedModule):
    def __init__(self, cfg):
        super().__init__()
        self.safetycost = SafetyCost(cfg)
        self.headwaycost = HeadwayCost(cfg)
        self.lrdividercost = LR_divider(cfg)
        self.comfortcost = Comfort(cfg)
        self.progresscost = Progress(cfg)
        self.rulecost = Rule(cfg)
        self.costvolume = Cost_Volume(cfg)
        self.n_future = cfg.N_FUTURE_FRAMES
        H, W = (int(v) for v in self.safetycost.bev_dimension[:2])
        if H != W:
            raise NotImplementedError(f"Cost_Function on a {H} x {W} grid: the reference's Rule and HeadwayCost view the "
                                      "map as (W, H) (cost.py:195,255), so only square grids have a defined meaning")

    def _pack(self):
        """Host values of the call descriptor, read once per parameter version (the footprints and SafetyCost.w)."""
        s = self.safetycost
        dx, bx = s.dx.detach().cpu(), s.bx.detach().cpu()
        lam = int(s._lambda / dx[0])          # cost.py:110: metres -> cells in fp32, then used as metres (kept as is)
        H, W = (int(v) for v in s.bev_dimension[:2])
        return dict(H=H, W=W, dx=dx.tolist(), bx=bx.tolist(), fp0=footprint(s.W, s.H, dx, bx, 0),
                    fp1=footprint(s.W, s.H, dx, bx, lam), safety=float(s.factor),
                    headway=float(self.headwaycost.factor), lrdivider=float(self.lrdividercost.factor),
                    comfort=float(self.comfortcost.factor), progress=float(self.progresscost.factor),
                    volume=float(self.costvolume.factor), rule=float(self.rulecost.factor),
                    safety_w=s.w.detach().cpu().tolist(),
                    headway_dist=float(self.headwaycost.L), lane_dist=float(self.lrdividercost.L))

    def desc(self, B, N, T, n_hd, traj_c, G=0):
        return ops.plan_desc(B=B, N=N, T=T, n_hd=n_hd, traj_c=traj_c, G=G, **self.packed())

    def forward(self, cost_volume, trajs, semantic_pred, lane_divider, drivable_area, target_point):
        """cost_volume (B, T, H, W), trajs (B, N, T, 2) [or (B, N, T, 3), the third component ignored], semantic_pred
        (B, T, H, W) bool, lane_divider / drivable_area (B, 1 or 2, H, W), target_point (B, 2) -> cost_fc (B, N),
        cost_fo (B, N, T), fp32 on the device."""
        if lane_divider.ndim != 4 or drivable_area.ndim != 4 or lane_divider.shape[1] != drivable_area.shape[1] or \
                lane_divider.shape[1] not in (1, 2):
            raise ValueError("lane_divider and drivable_area: (B, 1, H, W) raw maps or (B, 2, H, W) logits, both alike "
                             f"(got {tuple(lane_divider.shape)} and {tuple(drivable_area.shape)})")
        B, N, T, c = trajs.shape
        d = self.desc(B, N, T, lane_divider.shape[1], c)
        return ops.plan_cost(d, trajs, semantic_pred, cost_volume, target_point, lane_divider, drivable_area)
