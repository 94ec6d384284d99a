"""Python entry points over the C ABI: tensors in, tensors out, current CUDA stream, no fallback."""
import ctypes
from typing import Optional

import torch

from . import _lib


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("stp3_b200 ops run on CUDA tensors only (there is no CPU path)")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def _host3(v):
    a = torch.as_tensor(v, dtype=torch.float32, device="cpu").reshape(3)
    return (ctypes.c_float * 3)(*[float(x) for x in a])   # exact: a python float holds every fp32


class Workspace:
    """Grow-only device scratch buffer reused between calls (the lift-splat's L2-resident scatter grid)."""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None

    def get(self, nbytes: int, device) -> torch.Tensor:
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
            self.reset()
        return self.buf

    def reset(self):
        """Zero the buffer (required once after allocation, and after any failed call; see include/stp3_b200.h)."""
        if self.buf is not None:
            with torch.cuda.device(self.buf.device):
                code = _lib.lib().stp3_lift_splat_workspace_init(
                    self.buf.data_ptr(), self.buf.numel(), torch.cuda.current_stream(self.buf.device).cuda_stream)
            _lib.check(code, "stp3_lift_splat_workspace_init")


_default_ws = Workspace()


def _ptr(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def _lift_desc(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim, discount=0.0,
               feat_channels_last=False, use_depth_distribution=True, f_begin=0, f_count=0):
    """What every lift-splat call shares: the shapes, fp32 contiguous inputs on feat's device, the shape checks and the
    stp3_lift_splat_desc (include/stp3_b200.h).  Returns (desc, feat, depth_logits); desc.keep holds the geometry
    tensors the descriptor points into, so they live as long as it does."""
    _require_cuda(feat, depth_logits)
    dev = feat.device
    if feat_channels_last:
        B, S, N, Hf, Wf, C = feat.shape
    else:
        B, S, N, C, Hf, Wf = feat.shape
    D = ds.numel()
    nx, ny, nz = (int(v) for v in bev_dim)
    feat = _f32c(feat)
    depth_logits = _f32c(depth_logits) if depth_logits is not None else None
    if use_depth_distribution:
        assert depth_logits is not None and tuple(depth_logits.shape) == (B, S, N, D, Hf, Wf), "depth_logits shape"
    geom = [_f32c(t.to(dev)) for t in (cam_M, cam_t, ego_R, ego_t, xs, ys, ds)]
    cam_M, cam_t, ego_R, ego_t, xs, ys, _ = geom
    assert cam_M.shape == (B, S, N, 3, 3) and cam_t.shape == (B, S, N, 3)
    assert ego_R.shape == (B, S, 3, 3) and ego_t.shape == (B, S, 3)
    assert xs.numel() == Wf and ys.numel() == Hf
    desc = _lib.LiftSplatDesc(*(t.data_ptr() for t in geom), _host3(bev_off), _host3(bev_res), nx, ny, nz,
                              float(discount), B, S, N, D, Hf, Wf, C, int(feat_channels_last),
                              int(use_depth_distribution), int(f_begin), int(f_count))
    desc.keep = geom
    return desc, feat, depth_logits


def _lift_fwd(desc, feat, depth_logits, workspace: Optional[Workspace], out, out_layout: int, ranks=None, psum=None,
              peer_ptrs=None):
    """stp3_lift_splat_fwd on the current stream -- or, when torch.are_deterministic_algorithms_enabled() (warn_only
    included), its fixed-point form stp3_lift_splat_fwd_det, whose results are bitwise repeatable.  A CUDA graph
    replays the mode it was captured in.  The workspace is re-initialised when the call fails."""
    L = _lib.lib()
    dev = feat.device
    workspace = workspace or _default_ws
    det = torch.are_deterministic_algorithms_enabled()
    name = "stp3_lift_splat_fwd_det" if det else "stp3_lift_splat_fwd"
    nbytes = L.stp3_lift_splat_det_workspace_bytes(desc) if det else L.stp3_lift_splat_workspace_bytes(desc)
    ws = workspace.get(nbytes, dev)
    peers = (ctypes.c_void_p * len(peer_ptrs))(*[int(x) for x in peer_ptrs]) if peer_ptrs is not None else None
    with torch.cuda.device(dev):
        code = getattr(L, name)(desc, feat.data_ptr(), _ptr(depth_logits), _ptr(ranks), _ptr(psum), ws.data_ptr(),
                                ws.numel(), _ptr(out), out_layout, len(peer_ptrs or ()), peers,
                                torch.cuda.current_stream(dev).cuda_stream)
    if code != 0:
        workspace.reset()
    _lib.check(code, name)


def lift_splat(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
               discount: float, *, feat_channels_last: bool = False, out_channels_last: bool = False,
               use_depth_distribution: bool = True, return_ranks: bool = False, pool_sum: bool = False,
               workspace: Optional[Workspace] = None, out: Optional[torch.Tensor] = None,
               out_hilo: Optional[torch.Tensor] = None):
    """Fused lift (softmax-depth (x) context) + ego-aligned voxel pooling + temporal discount.

      feat          (B,S,N,C,Hf,Wf) or, with feat_channels_last, (B,S,N,Hf,Wf,C)
      depth_logits  (B,S,N,D,Hf,Wf)
      cam_M/cam_t/ego_R/ego_t/xs/ys/ds  see utils.geometry.lift_matrices / frustum_axes
      bev_off, bev_res (3,) float (host values); bev_dim (3,) int
    Returns out (B,S,C,X,Y) [or (B,S,X,Y,C)], and optionally ranks (B,S,N,D,Hf,Wf) int32 and pool sums (B,S,C).
    Semantics: stp3/models/stp3.py:186-301 of the reference."""
    desc, feat, depth_logits = _lift_desc(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res,
                                          bev_dim, discount, feat_channels_last, use_depth_distribution)
    dev = feat.device
    B, S, C, nx, ny = desc.B, desc.S, desc.C, desc.nx, desc.ny
    oshape = (B, S, nx, ny, C) if out_channels_last else (B, S, C, nx, ny)
    layout = int(out_channels_last)
    if out_hilo is not None:      # two bf16 planes (2,B,S,nx,ny,C): the activation format of the tensor-core path
        assert tuple(out_hilo.shape) == (2, B, S, nx, ny, C) and out_hilo.dtype == torch.bfloat16 and out_hilo.is_contiguous()
        out, layout = out_hilo, 2
    elif out is None:
        out = torch.empty(oshape, dtype=torch.float32, device=dev)
    else:
        assert tuple(out.shape) == oshape and out.is_contiguous() and out.dtype == torch.float32
    ranks = torch.empty((B, S, desc.N, desc.D, desc.Hf, desc.Wf), dtype=torch.int32, device=dev) if return_ranks else None
    psum = torch.zeros((B, S, C), dtype=torch.float32, device=dev) if pool_sum else None
    _lift_fwd(desc, feat, depth_logits, workspace, out, layout, ranks=ranks, psum=psum)
    res = (out,)
    if return_ranks:
        res += (ranks,)
    if pool_sum:
        res += (psum,)
    return res if len(res) > 1 else out


def lift_splat_plan(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
                    discount: float, *, feat_channels_last: bool = False, out_channels_last: bool = False,
                    use_depth_distribution: bool = True, return_ranks: bool = False, pool_sum: bool = False,
                    workspace: Optional[Workspace] = None, out: Optional[torch.Tensor] = None,
                    out_hilo: Optional[torch.Tensor] = None, f_begin: int = 0, f_count: int = 0, n_peers: int = 0) -> dict:
    """The kernels lift_splat() (or, with f_count > 0, lift_splat_frames()) launches for these arguments:
    stp3_lift_splat_plan (include/stp3_b200.h) as a dict of its fields.  Launches nothing.  return_ranks, pool_sum,
    workspace and out do not change the plan; they are accepted so that lift_splat()'s arguments can be passed as they
    are."""
    desc, feat, depth_logits = _lift_desc(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res,
                                          bev_dim, discount, feat_channels_last, use_depth_distribution, f_begin, f_count)
    layout = 2 if out_hilo is not None else 1 if (out_channels_last or f_count > 0) else 0
    plan = _lib.LiftSplatPlan()
    code = _lib.lib().stp3_lift_splat_plan(desc, feat.data_ptr(), _ptr(depth_logits), layout, int(n_peers),
                                           ctypes.byref(plan))
    _lib.check(code, "stp3_lift_splat_plan")
    return {name: getattr(plan, name) for name, _ in _lib.LiftSplatPlan._fields_}


def lift_splat_backward(grad_out, feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
                        discount: float, *, use_depth_distribution: bool = True, feat_channels_last: bool = False):
    """Gradients of lift_splat()'s (B,S,C,X,Y) output w.r.t. feat (B,S,N,C,Hf,Wf) and depth_logits (B,S,N,D,Hf,Wf):
    stp3_lift_splat_bwd (include/stp3_b200.h).  With feat_channels_last feat and its gradient are (B,S,N,Hf,Wf,C)
    (stp3_lift_splat_bwd_cl: the same values, no transposes).  Returns (grad_feat, grad_depth_logits or None)."""
    desc, feat, depth_logits = _lift_desc(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res,
                                          bev_dim, discount, feat_channels_last, use_depth_distribution)
    dev = feat.device
    grad_out = _f32c(grad_out)
    assert tuple(grad_out.shape) == (desc.B, desc.S, desc.C, desc.nx, desc.ny)
    L = _lib.lib()
    nbytes = L.stp3_lift_splat_bwd_scratch_bytes(desc)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    g_feat = torch.empty_like(feat)
    g_depth = torch.empty_like(depth_logits) if (use_depth_distribution and depth_logits is not None) else None
    name = "stp3_lift_splat_bwd_cl" if feat_channels_last else "stp3_lift_splat_bwd"
    with torch.cuda.device(dev):
        code = getattr(L, name)(desc, grad_out.data_ptr(), feat.data_ptr(), _ptr(depth_logits), scratch.data_ptr(),
                                nbytes, g_feat.data_ptr(), _ptr(g_depth), torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(code, name)
    return g_feat, g_depth


class LiftSplatFunction(torch.autograd.Function):
    """Differentiable lift-splat: forward = stp3_lift_splat_fwd, backward = stp3_lift_splat_bwd (stp3_lift_splat_bwd_cl
    for channels-last feat, whose gradient comes back in that layout).  Gradients flow to the
    context features and the depth logits; calibration, ego-motion and the integer voxel indices carry none (like the
    reference, whose indices pass through .long(), stp3.py:289)."""

    @staticmethod
    def forward(ctx, feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim, discount,
                use_depth_distribution, workspace, feat_channels_last=False):
        out = lift_splat(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim, discount,
                         use_depth_distribution=use_depth_distribution, workspace=workspace,
                         feat_channels_last=feat_channels_last)
        ctx.save_for_backward(feat, depth_logits if depth_logits is not None else feat.new_empty(0),
                              cam_M, cam_t, ego_R, ego_t, xs, ys, ds)
        ctx.host = (bev_off, bev_res, bev_dim, discount, use_depth_distribution, depth_logits is not None,
                    feat_channels_last)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds = ctx.saved_tensors
        bev_off, bev_res, bev_dim, discount, use_dd, has_depth, feat_cl = ctx.host
        g_feat, g_depth = lift_splat_backward(grad_out, feat, depth_logits if has_depth else None, cam_M, cam_t, ego_R,
                                              ego_t, xs, ys, ds, bev_off, bev_res, bev_dim, discount,
                                              use_depth_distribution=use_dd, feat_channels_last=feat_cl)
        return (g_feat, g_depth) + (None,) * 14


def lift_splat_autograd(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
                        discount: float, *, use_depth_distribution: bool = True, workspace: Optional[Workspace] = None,
                        feat_channels_last: bool = False):
    """lift_splat() ((B,S,C,X,Y) out; feat NCHW like the reference, or (B,S,N,Hf,Wf,C) with feat_channels_last) with
    gradients to feat, in its own layout, and depth_logits."""
    return LiftSplatFunction.apply(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
                                   float(discount), bool(use_depth_distribution), workspace, bool(feat_channels_last))


def lift_splat_frames(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res, bev_dim,
                      f_begin: int, f_count: int, *, feat_channels_last: bool = False,
                      use_depth_distribution: bool = True, workspace: Optional[Workspace] = None,
                      peer_ptrs=None) -> Optional[torch.Tensor]:
    """Frame-sharded lift-splat: RAW (no discount recurrence) channels-last splats (f_count, X, Y, C) fp32 of the flat
    frames f_begin + [0, f_count), f = b*S + t.  See the frame-sharded mode of stp3_lift_splat_fwd in
    include/stp3_b200.h.  peer_ptrs (list of device pointers, one (B*S, X, Y, C) fp32 buffer per rank): the finalize
    epilogue stores the frames into slot f of every rank's buffer instead; returns None."""
    if f_count <= 0:        # f_count == 0 would describe the unsharded call
        raise RuntimeError(f"lift_splat_frames: empty frame range (f_count={f_count})")
    desc, feat, depth_logits = _lift_desc(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, bev_off, bev_res,
                                          bev_dim, 0.0, feat_channels_last, use_depth_distribution, f_begin, f_count)
    out = None
    if peer_ptrs is None:
        out = torch.empty((f_count, desc.nx, desc.ny, desc.C), dtype=torch.float32, device=feat.device)
    _lift_fwd(desc, feat, depth_logits, workspace, out, 1, peer_ptrs=peer_ptrs)
    return out


def bev_discount(raw: torch.Tensor, discount: float) -> torch.Tensor:
    """raw (B,S,X,Y,C) fp32 channels-last per-frame splats -> (2,B,S,X,Y,C) bf16 hi/lo planes of
    out[t] = out[t-1]*discount + raw[t]  (stp3.py:296)."""
    _require_cuda(raw)
    raw = _f32c(raw)
    B, S, X, Y, C = raw.shape
    planes = torch.empty((2, B, S, X, Y, C), dtype=torch.bfloat16, device=raw.device)
    with torch.cuda.device(raw.device):
        code = _lib.lib().stp3_bev_discount(raw.data_ptr(), B, S, X, Y, C, float(discount), planes[0].data_ptr(),
                                            planes[1].data_ptr(), torch.cuda.current_stream(raw.device).cuda_stream)
    _lib.check(code, "stp3_bev_discount")
    return planes


# ------------------------------------------------------------------------------------------------ planning (eval)
def plan_desc(*, B, N, T, H, W, dx, bx, fp0, fp1, safety, headway, lrdivider, comfort, progress, volume, rule, safety_w,
              headway_dist, lane_dist, n_hd, traj_c, G=0) -> "_lib.PlanDesc":
    """stp3_plan_desc (include/stp3_b200.h) from host values; dx, bx, safety_w are pairs of fp32 values, fp0 / fp1 the
    footprints as (first row, last row, first column, last column)."""
    F2, I4 = ctypes.c_float * 2, ctypes.c_int * 4
    return _lib.PlanDesc(B=B, N=N, T=T, H=H, W=W, dx=F2(*map(float, dx)), bx=F2(*map(float, bx)), fp0=I4(*fp0),
                         fp1=I4(*fp1), safety=safety, headway=headway, lrdivider=lrdivider, comfort=comfort,
                         progress=progress, volume=volume, rule=rule, safety_w=F2(*map(float, safety_w)), headway_dist=headway_dist,
                         lane_dist=lane_dist, n_hd=n_hd, traj_c=traj_c, G=G)


def _shape(t: torch.Tensor, shape, what: str):
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what}: expected shape {tuple(shape)}, got {tuple(t.shape)}")


def plan_cost(desc, trajs, occupancy, cost_volume, target_points, lane, drivable):
    """Cost_Function.forward (cost.py:25-46) on the device: trajs (B, N, T, traj_c) fp32, occupancy (B, T, H, W) bool,
    cost_volume (B, T, H, W), target_points (B, 2), lane / drivable (B, n_hd, H, W) -> cost_fc (B, N), cost_fo (B, N, T)
    fp32.  Two launches (stp3_plan_maps, stp3_plan_cost), no host synchronisation."""
    _require_cuda(trajs, occupancy, cost_volume, target_points, lane, drivable)
    B, N, T, H, W = desc.B, desc.N, desc.T, desc.H, desc.W
    dev = trajs.device
    if occupancy.dtype != torch.bool:
        raise TypeError(f"semantic_pred must be a bool occupancy map (got {occupancy.dtype}): the footprint sums count "
                        "occupied cells")
    _shape(trajs, (B, N, T, desc.traj_c), "trajs")
    _shape(occupancy, (B, T, H, W), "semantic_pred")
    _shape(cost_volume, (B, T, H, W), "cost_volume")
    _shape(target_points, (B, 2), "target_points")
    _shape(lane, (B, desc.n_hd, H, W), "lane_divider")
    _shape(drivable, (B, desc.n_hd, H, W), "drivable_area")
    trajs, cost_volume, target_points, lane, drivable = (_f32c(t) for t in (trajs, cost_volume, target_points, lane,
                                                                              drivable))
    occ = occupancy.contiguous().view(torch.uint8)
    drv = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    dang = torch.empty((B, H, W), dtype=torch.uint8, device=dev)
    lane_cost = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    fc = torch.empty((B, N), dtype=torch.float32, device=dev)
    fo = torch.empty((B, N, T), dtype=torch.float32, device=dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.stp3_plan_maps(desc, lane.data_ptr(), drivable.data_ptr(), drv.data_ptr(), dang.data_ptr(),
                                    lane_cost.data_ptr(), st), "stp3_plan_maps")
        _lib.check(L.stp3_plan_cost(desc, trajs.data_ptr(), occ.data_ptr(), cost_volume.data_ptr(),
                                    target_points.data_ptr(), drv.data_ptr(), dang.data_ptr(), lane_cost.data_ptr(),
                                    fc.data_ptr(), fo.data_ptr(), st), "stp3_plan_cost")
    return fc, fo


def plan_refine(desc, windows_host, windows, trajs, cost_fc, cost_fo, h0, target_points, w_ih, b_ih, w_hh_t, b_hh,
                w1_t, b1, w2, b2):
    """The selection and GRU refinement of Planning.forward (planning_model.py:129-145): windows (B, 2) int32 (first
    candidate, count) on the device and the same values on the host (windows_host, checked before the launch) ->
    output_traj (B, T, 3) fp32 and the selected candidate index (B,) int32."""
    _require_cuda(windows, trajs, cost_fc, cost_fo, h0)
    B, N, T, G = desc.B, desc.N, desc.T, desc.G
    dev = trajs.device
    if windows_host.dtype != torch.int32 or windows.dtype != torch.int32 or windows_host.is_cuda:
        raise TypeError("windows: int32, one copy on the host and one on the device")
    _shape(windows_host, (B, 2), "windows_host")
    _shape(windows, (B, 2), "windows")
    _shape(trajs, (B, N, T, desc.traj_c), "trajs")
    _shape(cost_fc, (B, N), "cost_fc")
    _shape(cost_fo, (B, N, T), "cost_fo")
    _shape(h0, (B, G), "h0")
    _shape(w_hh_t, (G, 3 * G), "w_hh_t")
    _shape(w1_t, (G, G), "w1_t")
    windows_host, windows = windows_host.contiguous(), windows.contiguous()
    trajs, cost_fc, cost_fo, h0, target_points = (_f32c(t) for t in (trajs, cost_fc, cost_fo, h0, target_points))
    out = torch.empty((B, T, 3), dtype=torch.float32, device=dev)
    sel = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_plan_refine(desc, windows_host.data_ptr(), windows.data_ptr(), trajs.data_ptr(),
                                           cost_fc.data_ptr(), cost_fo.data_ptr(), h0.data_ptr(),
                                           target_points.data_ptr(), w_ih.data_ptr(), b_ih.data_ptr(),
                                           w_hh_t.data_ptr(), b_hh.data_ptr(), w1_t.data_ptr(), b1.data_ptr(),
                                           w2.data_ptr(), b2.data_ptr(), out.data_ptr(), sel.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(code, "stp3_plan_refine")
    return out, sel
