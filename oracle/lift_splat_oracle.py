"""ORACLE (test infrastructure, not product code) — CPU restatement of ST-P3's lift-splat.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this file.  The product package (stp3_b200/) never does.

Restates, in numpy with every fp32 rounding step written out explicitly:

  * frustum axes                  stp3/models/stp3.py:111-130
  * camera->ego geometry          stp3/models/stp3.py:186-201
  * softmax(depth) (x) context    stp3/models/stp3.py:215-216
  * sequential ego-motion warp    stp3/models/stp3.py:270-277
  * voxel index (div + trunc)     stp3/models/stp3.py:287-289
  * in-bounds mask and rank       stp3/models/stp3.py:239-255
  * per-pillar sum                stp3/utils/geometry.py:299-318 (VoxelsSumming)
  * discount recurrence + layout  stp3/models/stp3.py:292-299
  * BEV grid parameters           stp3/utils/geometry.py:40-59
  * 6-DoF pose -> 4x4             stp3/utils/geometry.py:124-172

Parity pinning: the reference ships NO tests, golden vectors or fixtures for this path
(SURVEY.md §4/§8c), so the oracle is pinned against outputs of the reference itself, run in the
build container through oracle/ref_loader.py; the results are committed under tests/golden/ by
oracle/make_golden.py and re-checked by tests/test_oracle_vs_golden.py.  Geometry and voxel
indices are compared BITWISE; pooled features are compared in fp64 because the reference's fp32
cumsum-trick is itself only accurate to ~3e-3 relative (SURVEY.md headline fact 6).

fp32 op order (verified against the reference's CPU matmul, 0 mismatching floats):
    p = ((m0*x + m1*y) + m2*z) + t      every * and + individually rounded to fp32, no FMA.
"""
import numpy as np

F32 = np.float32


# ----------------------------------------------------------------------------- host-side parameters
def bev_params(x_bound, y_bound, z_bound):
    """geometry.py:40-59.  torch.tensor(list of python floats) rounds the *double* expression
    `min + step/2` to fp32 once; dimension is the double quotient truncated to int64."""
    rows = [x_bound, y_bound, z_bound]
    res = np.array([r[2] for r in rows], dtype=np.float64).astype(F32)
    start = np.array([r[0] + r[2] / 2.0 for r in rows], dtype=np.float64).astype(F32)
    dim = np.array([int((r[1] - r[0]) / r[2]) for r in rows], dtype=np.int64)
    return res, start, dim


def bev_offset(res, start):
    """stp3.py:288: (bev_start_position - bev_resolution / 2.0) evaluated in fp32."""
    return (start - (res / F32(2.0)).astype(F32)).astype(F32)


def frustum_axes(final_dim, downsample, d_bound):
    """stp3.py:111-130.  The reference builds the axes with torch.linspace / torch.arange on the CPU at
    model construction.  ATen's vectorised linspace kernel rounds differently depending on the host ISA
    (AVX2 vs AVX-512 chunking), so the axes are treated as HOST PARAMETERS: obtained with the very same
    torch calls and handed to the restatement (and to the CUDA kernel) as three small arrays; the golden
    fixtures carry the build container's values."""
    import torch
    h, w = final_dim
    hf, wf = h // downsample, w // downsample
    xs = torch.linspace(0, w - 1, wf, dtype=torch.float).numpy()
    ys = torch.linspace(0, h - 1, hf, dtype=torch.float).numpy()
    ds = torch.arange(*d_bound, dtype=torch.float).numpy()
    return xs, ys, ds


def host_matrices(intrinsics, extrinsics, future_egomotion):
    """Host parameters exactly as the reference evaluates them (torch calls, not restated because LAPACK
    inverse / vectorised sin-cos are library-defined):
      cam_M = R . inverse(K) (stp3.py:190,196), cam_t (stp3.py:190,198),
      ego R|t = Rx.Ry.Rz | (tx,ty,tz)  (geometry.py:124-172, stp3.py:234-235)."""
    import torch
    K = torch.as_tensor(intrinsics)
    E = torch.as_tensor(extrinsics)
    ego = torch.as_tensor(future_egomotion)
    cam_M = E[..., :3, :3].matmul(torch.inverse(K))
    cam_t = E[..., :3, 3]
    ang = ego[..., 3:].reshape(-1, 3)
    x, y, z = ang[:, 0], ang[:, 1], ang[:, 2]
    o, zz = torch.ones_like(z), torch.zeros_like(z)
    zm = torch.stack([torch.cos(z), -torch.sin(z), zz, torch.sin(z), torch.cos(z), zz, zz, zz, o], 1).view(-1, 3, 3)
    ym = torch.stack([torch.cos(y), zz, torch.sin(y), zz, o, zz, -torch.sin(y), zz, torch.cos(y)], 1).view(-1, 3, 3)
    xm = torch.stack([o, zz, zz, zz, torch.cos(x), -torch.sin(x), zz, torch.sin(x), torch.cos(x)], 1).view(-1, 3, 3)
    R = xm.bmm(ym).bmm(zm).view(*ego.shape[:-1], 3, 3)
    return (cam_M.contiguous().numpy(), cam_t.contiguous().numpy(), R.contiguous().numpy(),
            ego[..., :3].contiguous().numpy())


# ----------------------------------------------------------------------------- geometry
def _affine(m, t, x, y, z):
    """((m0*x + m1*y) + m2*z) + t with separate fp32 roundings; m (3,3), t (3,), x/y/z arrays."""
    out = []
    for r in range(3):
        a = (m[r, 0] * x).astype(F32)
        b = (m[r, 1] * y).astype(F32)
        c = (m[r, 2] * z).astype(F32)
        s = ((a + b).astype(F32) + c).astype(F32)
        out.append((s + t[r]).astype(F32))
    return out


def geometry(cam_M, cam_t, xs, ys, ds):
    """stp3.py:186-201 for ONE (b,t): cam_M (N,3,3) = R.K^-1, cam_t (N,3) -> (N,D,Hf,Wf,3) fp32."""
    n = cam_M.shape[0]
    D, Hf, Wf = len(ds), len(ys), len(xs)
    d = ds.reshape(D, 1, 1)
    px = (xs.reshape(1, 1, Wf) * d).astype(F32) * np.ones((1, Hf, 1), F32)
    py = (ys.reshape(1, Hf, 1) * d).astype(F32) * np.ones((1, 1, Wf), F32)
    pz = d * np.ones((1, Hf, Wf), F32)
    out = np.empty((n, D, Hf, Wf, 3), dtype=F32)
    for i in range(n):
        gx, gy, gz = _affine(cam_M[i], cam_t[i], px, py, pz)
        out[i, ..., 0], out[i, ..., 1], out[i, ..., 2] = gx, gy, gz
    return out


def ego_warp(geom, ego_R, ego_t):
    """stp3.py:270-277 for ONE sample: geom (S,N,D,Hf,Wf,3); frames 0..t are transformed by pose t,
    for t = 0..S-2, sequentially with an fp32 rounding after every step.  Returns a new array."""
    g = geom.copy()
    S = g.shape[0]
    for t in range(S - 1):
        x, y, z = g[: t + 1, ..., 0], g[: t + 1, ..., 1], g[: t + 1, ..., 2]
        nx, ny, nz = _affine(ego_R[t], ego_t[t], x, y, z)
        g[: t + 1, ..., 0], g[: t + 1, ..., 1], g[: t + 1, ..., 2] = nx, ny, nz
    return g


def voxel_index(geom, off, res, dim):
    """stp3.py:287-289 + 239-255.  Returns idx (…,3) int64 (trunc toward zero) and rank (…) int64 with
    -1 for points outside the grid.  Non-finite / huge values are masked (x86 cvttss2si gives
    INT64_MIN for them, which the reference's `>= 0` test rejects)."""
    q = ((geom - off).astype(F32) / res).astype(F32)
    ok = np.isfinite(q) & (np.abs(q) < F32(2.0 ** 62))
    idx = np.where(ok, np.trunc(np.where(ok, q, 0)), -1).astype(np.int64)
    keep = ok.all(-1)
    for a in range(3):
        keep &= (idx[..., a] >= 0) & (idx[..., a] < dim[a])
    rank = idx[..., 0] * (dim[1] * dim[2]) + idx[..., 1] * dim[2] + idx[..., 2]
    return idx, np.where(keep, rank, -1)


# ----------------------------------------------------------------------------- pooling
def softmax_depth(logits):
    """stp3.py:215 in fp64: logits (…,D,Hf,Wf) softmax over D."""
    z = logits.astype(np.float64)
    z = z - z.max(axis=-3, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=-3, keepdims=True)


def splat_frame(feat, prob, rank, nvox):
    """One (b,t) frame: feat (N,C,Hf,Wf) fp32, prob (N,D,Hf,Wf) fp64, rank (N,D,Hf,Wf) -> (C, nvox) fp64
    exact per-pillar sums of prob[n,d,h,w]*feat[n,c,h,w] (what VoxelsSumming approximates)."""
    N, C, Hf, Wf = feat.shape
    keep = rank >= 0
    r = rank[keep]
    p = prob[keep]
    n_i, d_i, h_i, w_i = np.nonzero(keep)
    out = np.zeros((C, nvox), dtype=np.float64)
    f64 = feat.astype(np.float64)
    for c in range(C):
        out[c] = np.bincount(r, weights=p * f64[n_i, c, h_i, w_i], minlength=nvox)
    return out


def lift_splat(feat, depth_logits, cam_M, cam_t, ego_R, ego_t, xs, ys, ds, off, res, dim, discount,
               use_depth_distribution=True):
    """Whole path for a batch.
      feat (B,S,N,C,Hf,Wf) f32, depth_logits (B,S,N,D,Hf,Wf) f32, cam_M (B,S,N,3,3), cam_t (B,S,N,3),
      ego_R (B,S,3,3), ego_t (B,S,3).
    Returns dict(bev=(B,S,C,X,Y) f64, rank=(B,S,N,D,Hf,Wf) int32 (-1 = masked), geom=(B,S,N,D,Hf,Wf,3) f32)."""
    B, S, N, C, Hf, Wf = feat.shape
    D = len(ds)
    X, Y, Z = int(dim[0]), int(dim[1]), int(dim[2])
    assert Z == 1, "the reference's squeeze(0) at stp3.py:298 assumes one height bin"
    bev = np.zeros((B, S, C, X, Y), dtype=np.float64)
    ranks = np.empty((B, S, N, D, Hf, Wf), dtype=np.int32)
    geoms = np.empty((B, S, N, D, Hf, Wf, 3), dtype=F32)
    if use_depth_distribution:
        prob = softmax_depth(depth_logits)
    else:  # stp3.py:218: features repeated over depth
        prob = np.ones(depth_logits.shape[:3] + (D, Hf, Wf), dtype=np.float64)
    for b in range(B):
        g = np.stack([geometry(cam_M[b, t], cam_t[b, t], xs, ys, ds) for t in range(S)])
        g = ego_warp(g, ego_R[b], ego_t[b])
        geoms[b] = g
        _, rank = voxel_index(g, off, res, dim)
        ranks[b] = rank
        acc = np.zeros((C, X * Y), dtype=np.float64)
        for t in range(S):
            acc = acc * np.float64(F32(discount)) + splat_frame(feat[b, t], prob[b, t], rank[t], X * Y * Z)
            bev[b, t] = acc.reshape(C, X, Y)
    return {"bev": bev, "rank": ranks, "geom": geoms}


# ----------------------------------------------------------------------------- backward (SURVEY.md row f2)
def lift_splat_backward(grad_bev, feat, depth_logits, rank, discount, use_depth_distribution=True):
    """fp64 gradients of loss w.r.t. feat and depth_logits given grad_bev = dloss/dbev (B,S,C,X,Y), restating the
    reference's autograd chain:
      discount recurrence bev[t] = bev[t-1]*discount + splat[t]   (stp3.py:296)  -> g_splat[t'] = sum_{t>=t'} discount^(t-t') g_bev[t]
      index_put / mask / sort / VoxelsSumming.backward            (stp3.py:239-295, geometry.py:321-330): every kept point
                                                                  receives the gradient row of its pillar, masked points zero
      outer product x = prob (x) feat                             (stp3.py:216)
      softmax over depth                                          (stp3.py:215)
    rank (B,S,N,D,Hf,Wf): pillar of every point, -1 = masked (from lift_splat())."""
    B, S, N, C, Hf, Wf = feat.shape
    nvox = grad_bev.shape[-1] * grad_bev.shape[-2]
    g = grad_bev.astype(np.float64).reshape(B, S, C, nvox)
    disc = np.float64(F32(discount))
    gs = np.zeros_like(g)
    for t in range(S - 1, -1, -1):
        gs[:, t] = g[:, t] + (gs[:, t + 1] * disc if t + 1 < S else 0.0)
    prob = softmax_depth(depth_logits) if use_depth_distribution else np.ones(rank.shape, dtype=np.float64)
    f64 = feat.astype(np.float64)
    g_feat = np.zeros(feat.shape, dtype=np.float64)
    g_prob = np.zeros(rank.shape, dtype=np.float64)
    for b in range(B):
        for t in range(S):
            r = rank[b, t]                                          # (N,D,Hf,Wf)
            keep = r >= 0
            gp = np.where(keep[None], gs[b, t][:, np.where(keep, r, 0)], 0.0)      # (C,N,D,Hf,Wf) gradient of every point
            g_feat[b, t] = np.einsum('cndhw,ndhw->nchw', gp, prob[b, t])
            g_prob[b, t] = np.einsum('cndhw,nchw->ndhw', gp, f64[b, t])
    if not use_depth_distribution:
        return g_feat, None
    dot = (prob * g_prob).sum(axis=-3, keepdims=True)
    return g_feat, prob * (g_prob - dot)
