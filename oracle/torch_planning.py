"""ORACLE (test infrastructure) -- fp64 model of the eval-mode planner (stp3/models/planning_model.py, stp3/cost.py).

Only tests/ and tools/ may import this.  Every trajectory-derived index (the footprint cells of get_points, the cell of
discretize) is computed with the reference's fp32 tensor expressions, so boundaries fall where they fall in the
reference; every cost term, the softmaxes, the lane distance, the Bottlenecks, the GRU and the MLP are evaluated in
fp64.  Takes any module carrying the reference's parameter tree (the reference's Planning or stp3_b200's).

  footprint_cells(fp)                      the integer cells of a footprint (first row, last row, first col, last col)
  maps(lane, drivable)                     drivable probability, dangerous area, lane mask (fp64)
  cost_function(...)                       Cost_Function.forward -> (cost_fc (B, N), cost_fo (B, N, T)), fp64
  terms(...)                               the same, split into the seven clamped terms
  reduce_channel(cam_front, planning)      the four Bottlenecks, flattened (fp64)
  refine(h0, traj, target, planning)       the T GRUCell steps and the decoder (fp64)
  planning_forward(...)                    Planning.forward in eval -> (output_traj, selected index, cost_fc, cost_fo)
"""
import torch
import torch.nn.functional as F

from .torch_dense import _bn
from .torch_predict import _conv, maxpool2_pad


def footprint_cells(fp):
    r0, r1, c0, c1 = fp
    rr, cc = torch.meshgrid(torch.arange(r0, r1 + 1), torch.arange(c0, c1 + 1), indexing="ij")
    return torch.stack([rr.reshape(-1), cc.reshape(-1)], -1)          # (P, 2) int64, row-major


def get_points(trajs32, dx, rc, H, W):
    """cost.py:83-102 in fp32: trajs32 (B, N, T, 2) flipped fp32 points, dx fp32 (2,), rc (P, 2) int64 -> rows, cols
    (B, N, T, P) int64."""
    B, N, T, _ = trajs32.shape
    t = trajs32.view(B, N, T, 1, 2) / dx
    t = t[..., [1, 0]] + rc
    rr = torch.clamp(t[..., 0].long(), 0, H - 1)
    cc = torch.clamp(t[..., 1].long(), 0, W - 1)
    return rr, cc


def discretize(trajs32, dx, bx, H, W):
    """cost.py:125-140 in fp32: y with bx[0] / dx[0], x with bx[1] / dx[1]."""
    yi = torch.clamp(((trajs32[..., 1] - bx[0]) / dx[0]).long(), 0, H - 1)
    xi = torch.clamp(((trajs32[..., 0] - bx[1]) / dx[1]).long(), 0, W - 1)
    return yi, xi


def maps(lane, drivable):
    """lane / drivable (B, 1 or 2, H, W) -> drivable probability (B, H, W) fp64 (0 where < 0.5), dangerous area (B, H, W)
    bool, lane mask (B, H, W) bool (probability > 0.5, or the raw map's non-zero cells)."""
    if drivable.shape[1] == 2:
        drv = torch.softmax(drivable.double(), dim=1)[:, 1]
        drv = torch.where(drv < 0.5, torch.zeros_like(drv), drv)
    else:
        drv = drivable[:, 0].double()
    if lane.shape[1] == 2:
        lm = torch.softmax(lane.double(), dim=1)[:, 1] > 0.5
    else:
        lm = lane[:, 0] != 0
    return drv, drv == 0, lm


def lane_cost(lm, yi, xi, dx, L, factor):
    """LR_divider (cost.py:283-304) at the discretised cells: lm (B, H, W) bool, yi / xi (B, N, T) -> (B, N, T) fp64."""
    B = lm.shape[0]
    dx64 = dx.double()
    out = []
    for b in range(B):
        idx = torch.nonzero(lm[b])
        if len(idx) == 0:
            out.append(torch.zeros(yi.shape[1:], dtype=torch.float64))
            continue
        yx = torch.stack([yi[b], xi[b]], -1).unsqueeze(-2)                   # (N, T, 1, 2)
        d = ((yx - idx).double() * dx64.flip(0)).pow(2).sum(-1).sqrt().min(-1).values
        c = (L - d) ** 2
        out.append(torch.where(d > L, torch.zeros_like(c), c))
    return torch.stack(out) * factor


def terms(cf, cost_volume, trajs, semantic_pred, lane, drivable, target_points, fps):
    """The seven clamped terms of Cost_Function.forward (cost.py:34-41) in fp64.  cf: a module with the reference's
    Cost_Function children; fps: (footprint at lambda 0, footprint at lambda) as (r0, r1, c0, c1)."""
    s = cf.safetycost
    dx, bx = s.dx.detach().float().cpu(), s.bx.detach().float().cpu()
    H, W = (int(v) for v in s.bev_dimension[:2])
    t32 = trajs[..., :2].float().cpu() * torch.tensor([-1., 1.])
    t64 = t32.double()
    B, N, T, _ = t32.shape
    occ = semantic_pred.cpu().bool()
    drv, dang, lm = maps(lane.cpu(), drivable.cpu())
    bi = torch.arange(B).view(B, 1, 1, 1)
    ti = torch.arange(T).view(1, 1, T, 1)

    def area(m, pts, fp):                       # m (B, T, H, W) or (B, H, W): sum under the footprint
        rr, cc = get_points(pts, dx, footprint_cells(fp), H, W)
        return (m[bi, ti, rr, cc] if m.dim() == 4 else m[bi, rr, cc]).double().sum(-1)

    step = torch.cat([t64[:, :, :1], t64[:, :, 1:] - t64[:, :, :-1]], 2)
    vel = step.pow(2).sum(-1).sqrt() / 0.5
    w = s.w.detach().double().cpu()
    safety = (area(occ, t32, fps[0]) * w[0] + area(occ, t32, fps[1]) * vel * w[1]) * s.factor
    th = t32.clone()
    th[..., 1] = th[..., 1] + cf.headwaycost.L
    headway = area(occ.double() * drv[:, None], th, fps[0]) * cf.headwaycost.factor
    yi, xi = discretize(t32, dx, bx, H, W)
    lr = lane_cost(lm, yi, xi, dx, cf.lrdividercost.L, cf.lrdividercost.factor)
    cv = torch.clamp(cost_volume.double().cpu(), 0, 1000)[bi[..., 0], ti[..., 0], yi, xi] * cf.costvolume.factor
    rule = area(dang, t32, fps[0]) * cf.rulecost.factor
    # Comfort (cost.py:317-370)
    v_lat, v_lon = step[..., 0] / 0.5, step[..., 1] / 0.5
    zero = torch.zeros_like(v_lat[:, :, :1])
    a_lat = torch.cat([zero, (v_lat[:, :, 1:] - v_lat[:, :, :-1]) / 0.5], 2).abs().max(-1).values
    a_lon = torch.cat([zero, (v_lon[:, :, 1:] - v_lon[:, :, :-1]) / 0.5], 2).abs().max(-1).values
    acc = torch.cat([zero, (vel[:, :, 1:] - vel[:, :, :-1]) / 0.5], 2)
    jerk = torch.cat([zero, zero, (acc[:, :, 2:] - acc[:, :, 1:-1]) / 0.5], 2)[:, :, :T].abs().max(-1).values
    comfort = (torch.clamp(a_lat - 3, 0, 30) ** 2 + torch.clamp(a_lon - 3, 0, 30) ** 2 +
               torch.clamp(jerk - 1, 0, 20) ** 2) * cf.comfortcost.factor
    # Progress (cost.py:377-392)
    tp = target_points.double().cpu()
    far = 0 if tp.sum() < 0.5 else ((t64[:, :, -1] - tp[:, None]) ** 2).sum(-1)
    progress = (far - t64[..., 1].max(-1).values) * cf.progresscost.factor
    c = lambda v, lo=0.0: torch.clamp(v, lo, 100)
    return dict(safety=c(safety), headway=c(headway), lrdivider=c(lr), costvolume=c(cv), rule=c(rule),
                comfort=c(comfort), progress=c(progress, -100.0))


def cost_function(cf, cost_volume, trajs, semantic_pred, lane, drivable, target_points, fps):
    t = terms(cf, cost_volume, trajs, semantic_pred, lane, drivable, target_points, fps)
    return (t["comfort"] + t["progress"],
            t["safety"] + t["headway"] + t["lrdivider"] + t["costvolume"] + t["rule"])


def bottleneck(x, m):
    """Bottleneck in both built forms: downsampling (pad + pool on the skip) and projecting stride 1."""
    L = m.layers
    y = F.relu(_bn(_conv(x, L.conv_down_project), L.abn_down_project[0]))
    y = F.relu(_bn(_conv(y, L.conv), L.abn[0]))
    y = F.relu(_bn(_conv(y, L.conv_up_project), L.abn_up_project[0]))
    p = m.projection
    skip = maxpool2_pad(x) if hasattr(p, "upsample_skip_proj") else x
    return y + _bn(_conv(skip, p.conv_skip_proj), p.bn_skip_proj)


def reduce_channel(cam_front, planning):
    x = cam_front.double().cpu()
    for m in planning.reduce_channel:
        x = bottleneck(x, m)
    return x.flatten(1)


def refine(h0, traj, target_points, planning):
    """planning_model.py:132-145 in fp64: h0 (B, G), traj (B, T, >= 2) the selected trajectory, target (B, 2)."""
    g, d0, d2 = planning.GRU, planning.decoder[0], planning.decoder[2]
    W = lambda p: p.detach().double().cpu()
    h = h0.double().cpu()
    traj, tp = traj.double().cpu(), target_points.double().cpu()
    x = torch.zeros((h.shape[0], 2), dtype=torch.float64)
    out = []
    for i in range(traj.shape[1]):
        x = torch.cat([x, traj[:, i, :2], tp], -1)
        gi = x @ W(g.weight_ih).t() + W(g.bias_ih)
        gh = h @ W(g.weight_hh).t() + W(g.bias_hh)
        ir, iz, inn = gi.chunk(3, -1)
        hr, hz, hn = gh.chunk(3, -1)
        r, z = torch.sigmoid(ir + hr), torch.sigmoid(iz + hz)
        n = torch.tanh(inn + r * hn)
        h = (1 - z) * n + z * h
        x = F.relu(h @ W(d0.weight).t() + W(d0.bias)) @ W(d2.weight).t() + W(d2.bias)
        out.append(x)
    out = torch.stack(out, 1)
    return torch.cat([out, torch.zeros_like(out[..., :1])], -1)


def windows(commands, N):
    k = N // 3
    third = {'LEFT': (0, k), 'FORWARD': (k, k), 'RIGHT': (2 * k, N - 2 * k)}
    return [third.get(c, (0, N)) for c in commands]


def select(fc, fo, wins):
    """Index of the cheapest candidate (fp64 fc + sum fo) in each sample's window, lowest on ties, and the scores."""
    cs = fc + fo.sum(-1)
    sel = [s + int(torch.argmin(cs[b, s:s + c])) for b, (s, c) in enumerate(wins)]
    return torch.tensor(sel), cs


def planning_forward(planning, fps, cam_front, trajs, cost_volume, semantic_pred, hd_map, commands, target_points,
                     selected=None):
    """Planning.forward in eval (fp64).  `selected` (B,) overrides the fp64 argmin (to follow another implementation's
    choice among near-equal candidates).  Returns (output_traj, selected, cost_fc, cost_fo)."""
    if hd_map.shape[1] == 2:
        lane, drv = hd_map[:, 0:1], hd_map[:, 1:2]
    else:
        lane, drv = hd_map[:, 0:2], hd_map[:, 2:4]
    fc, fo = cost_function(planning.cost_function, cost_volume, trajs, semantic_pred, lane, drv, target_points, fps)
    sel, _ = select(fc, fo, windows(commands, trajs.shape[1]))
    if selected is not None:
        sel = torch.as_tensor(selected).long().cpu()
    h0 = reduce_channel(cam_front, planning)
    traj = trajs.cpu()[torch.arange(trajs.shape[0]), sel]
    return refine(h0, traj, target_points, planning), sel, fc, fo
