"""ORACLE / CPU BASELINE (test infrastructure) — op-for-op PyTorch restatement of the reference's CPU path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` leg may import this.

The reference is pure Python/PyTorch (SURVEY.md §0) and is not part of this repository (it need not
be present where bench.py runs), so the "reference arm" of bench.py times THIS port: it issues the same ATen operator sequence, with
the same materialised intermediates (17 MB geometry, 371 MB outer product, boolean-mask index, argsort, cumsum
trick, index_put, per-frame Python loops), as

    STP3.get_geometry                    stp3/models/stp3.py:186-201
    STP3.encoder_forward (softmax, (x))  stp3/models/stp3.py:214-221
    STP3.projection_to_birds_eye_view    stp3/models/stp3.py:226-301
    VoxelsSumming.forward                stp3/utils/geometry.py:299-318

tests/test_torch_port.py checks it against the golden vectors made from the real reference (bitwise on ranks via
the pooled output pattern, and to fp32 round-off on BEV values).  cpu_baseline.kind == "port".
"""
import torch


def frustum(xs, ys, ds):
    """(D,Hf,Wf,3) grid of (u, v, depth) (stp3.py:111-130), from the three axes."""
    D, Hf, Wf = ds.numel(), ys.numel(), xs.numel()
    return torch.stack((xs.view(1, 1, Wf).expand(D, Hf, Wf), ys.view(1, Hf, 1).expand(D, Hf, Wf),
                        ds.view(D, 1, 1).expand(D, Hf, Wf)), -1)


def get_geometry(frust, intrinsics, extrinsics):
    """intrinsics (M,N,3,3), extrinsics (M,N,4,4) -> (M,N,D,Hf,Wf,3)."""
    rot, trans = extrinsics[..., :3, :3], extrinsics[..., :3, 3]
    M, N, _ = trans.shape
    pts = frust.unsqueeze(0).unsqueeze(0).unsqueeze(-1)
    pts = torch.cat((pts[..., :2, :] * pts[..., 2:3, :], pts[..., 2:3, :]), 5)
    comb = rot.matmul(torch.inverse(intrinsics))
    pts = comb.view(M, N, 1, 1, 1, 3, 3).matmul(pts).squeeze(-1)
    pts += trans.view(M, N, 1, 1, 1, 3)
    return pts


def pose_matrix(vec):
    t = vec[..., :3].unsqueeze(-1)
    a = vec[..., 3:].contiguous().view(-1, 3)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    o, n = torch.ones_like(z), torch.zeros_like(z)
    zm = torch.stack([z.cos(), -z.sin(), n, z.sin(), z.cos(), n, n, n, o], 1).view(-1, 3, 3)
    ym = torch.stack([y.cos(), n, y.sin(), n, o, n, -y.sin(), n, y.cos()], 1).view(-1, 3, 3)
    xm = torch.stack([o, n, n, n, x.cos(), -x.sin(), n, x.sin(), x.cos()], 1).view(-1, 3, 3)
    R = xm.bmm(ym).bmm(zm).view(*vec.shape[:-1], 3, 3)
    T = torch.cat([R, t], -1)
    T = torch.nn.functional.pad(T, [0, 0, 0, 1], value=0)
    T[..., 3, 3] = 1.0
    return T


def cumsum_pool(x, geo, ranks):
    """VoxelsSumming.forward: prefix sums, keep the last row of every rank run, first differences."""
    x = x.cumsum(0)
    last = torch.ones(x.shape[0], dtype=torch.bool)
    last[:-1] = ranks[1:] != ranks[:-1]
    x, geo = x[last], geo[last]
    return torch.cat((x[:1], x[1:] - x[:-1])), geo


def projection(x, geometry, egomotion, bev_res, bev_start, bev_dim, discount):
    """x (B,S,N,D,Hf,Wf,C) [non-contiguous view, like the reference], geometry (B,S,N,D,Hf,Wf,3) mutated in place."""
    B, S, N, D, H, W, C = x.shape
    nx, ny, nz = (int(v) for v in bev_dim)
    out = torch.zeros((B, S, C, nx, ny), dtype=torch.float)
    pose = pose_matrix(egomotion)
    R, T = pose[..., :3, :3], pose[..., :3, 3]
    P = N * D * H * W
    for b in range(B):
        geo_b = geometry[b]
        for t in range(S - 1):
            g = R[b, t].view(1, 1, 1, 1, 1, 3, 3).matmul(geo_b[:t + 1].unsqueeze(-1)).squeeze(-1)
            g += T[b, t].view(1, 1, 1, 1, 1, 3)
            geo_b[:t + 1] = g
        bev = torch.zeros((nz, nx, ny, C))
        for t in range(S):
            xb = x[b, t].reshape(P, C)
            gi = ((geo_b[t] - (bev_start - bev_res / 2.0)) / bev_res).view(P, 3).long()
            keep = ((gi[:, 0] >= 0) & (gi[:, 0] < nx) & (gi[:, 1] >= 0) & (gi[:, 1] < ny)
                    & (gi[:, 2] >= 0) & (gi[:, 2] < nz))
            xb, gi = xb[keep], gi[keep]
            ranks = gi[:, 0] * (ny * nz) + gi[:, 1] * nz + gi[:, 2]
            order = ranks.argsort()
            xb, gi, ranks = xb[order], gi[order], ranks[order]
            xb, gi = cumsum_pool(xb, gi, ranks)
            cur = torch.zeros((nz, nx, ny, C))
            cur[gi[:, 2], gi[:, 0], gi[:, 1]] = xb
            bev = bev * discount + cur
            out[b, t] = bev.permute((0, 3, 1, 2)).squeeze(0)
    return out


def lift_splat(feat, depth_logits, intrinsics, extrinsics, egomotion, xs, ys, ds, bev_res, bev_start, bev_dim,
               discount):
    """feat (B,S,N,C,Hf,Wf), depth_logits (B,S,N,D,Hf,Wf) -> (B,S,C,X,Y), the reference's way."""
    B, S, N = feat.shape[:3]
    fr = frustum(xs, ys, ds)
    geo = get_geometry(fr, intrinsics.reshape(B * S, N, 3, 3), extrinsics.reshape(B * S, N, 4, 4))
    geo = geo.view(B, S, *geo.shape[1:])
    prob = depth_logits.reshape(B * S * N, *depth_logits.shape[3:]).softmax(dim=1)
    f = feat.reshape(B * S * N, *feat.shape[3:])
    x = prob.unsqueeze(1) * f.unsqueeze(2)
    x = x.view(B, S, N, *x.shape[1:]).permute(0, 1, 2, 4, 5, 6, 3)
    return projection(x, geo, egomotion, bev_res, bev_start, bev_dim, discount)
