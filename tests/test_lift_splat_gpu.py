"""GPU parity: the CUDA lift-splat (through the C ABI) against the oracle and the reference-made golden vectors.

Bars (BASELINE.md §5): voxel ranks bit-exact; BEV features within 1e-3 relative of the fp64 oracle (the kernel is
in fact ~1e-6: fp32 products, fp32 segment sums, fp32 atomics)."""
import numpy as np
import pytest
import torch

from oracle import lift_splat_oracle as O
from stp3_b200 import ops
from stp3_b200.utils import geometry as G
from stp3_b200.utils import synthetic as syn
from tests.helpers import LIFT_CASES, load_lift_case, sha

pytestmark = pytest.mark.gpu
REL_TOL = 1e-3     # north_star: BEV features within 1e-3 relative fp32


def run_cuda(cfg, inp, g, **kw):
    dev = torch.device("cuda:0")
    t = lambda a: torch.as_tensor(a).to(dev)
    return ops.lift_splat(inp["feat"].to(dev), inp["depth_logits"].to(dev), t(g["cam_M"]), t(g["cam_t"]),
                          t(g["ego_R"]), t(g["ego_t"]), t(g["xs"]), t(g["ys"]), t(g["ds"]),
                          g["bev_offset"], g["bev_resolution"], g["bev_dimension"], cfg.discount, **kw)


def run_oracle(cfg, inp, g, **kw):
    return O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), g["cam_M"], g["cam_t"], g["ego_R"],
                        g["ego_t"], g["xs"], g["ys"], g["ds"], g["bev_offset"], g["bev_resolution"],
                        g["bev_dimension"], cfg.discount, **kw)


def assert_bev_close(ours, oracle):
    ours = ours.astype(np.float64)
    scale = np.abs(oracle).max()
    diff = np.abs(ours - oracle)
    assert diff.max() <= 2e-5 * scale, (diff.max(), scale)
    big = np.abs(oracle) > 1e-3 * scale
    assert (diff[big] / np.abs(oracle[big])).max() <= REL_TOL
    # exactly-empty pillars stay exactly zero
    assert not np.any(ours[oracle == 0] != 0)


@pytest.mark.parametrize("name", LIFT_CASES)
def test_ranks_bit_exact_and_bev_close(name):
    cfg, inp, g = load_lift_case(name)
    out, ranks = run_cuda(cfg, inp, g, return_ranks=True)
    ora = run_oracle(cfg, inp, g)
    r = ranks.cpu().numpy()
    assert np.array_equal(r, ora["rank"]), f"{(r != ora['rank']).sum()} voxel ranks differ from the oracle"
    assert sha(r) == str(g["rank_sha"]), "voxel ranks differ from the reference's (golden fixture)"
    assert_bev_close(out.cpu().numpy(), ora["bev"])
    if "bev" in g:   # and directly against the reference's own fp32 output (its cumsum error is ~1e-4 of max)
        ref = g["bev"].astype(np.float64)
        assert np.abs(out.cpu().numpy() - ref).max() <= 3e-4 * np.abs(ref).max()


@pytest.mark.parametrize("name", ["tiny_randpose", "plumbing"])
def test_layout_variants(name):
    cfg, inp, g = load_lift_case(name)
    base = run_cuda(cfg, inp, g)
    inp_cl = dict(inp)
    inp_cl["feat"] = inp["feat"].permute(0, 1, 2, 4, 5, 3).contiguous()
    out_cl, psum = run_cuda(cfg, inp_cl, g, feat_channels_last=True, out_channels_last=True, pool_sum=True)
    a, b = base.cpu().numpy(), out_cl.permute(0, 1, 4, 2, 3).cpu().numpy()
    assert np.abs(a - b).max() <= 2e-5 * np.abs(a).max()          # atomics: summation order differs
    tot = base.double().sum(dim=(-1, -2)).cpu().numpy()
    assert np.allclose(psum.cpu().numpy(), tot, rtol=1e-4, atol=1e-4 * np.abs(tot).max())


def test_no_depth_distribution():
    cfg, inp, g = load_lift_case("tiny_level")
    out = run_cuda(cfg, inp, g, use_depth_distribution=False)
    ora = run_oracle(cfg, inp, g, use_depth_distribution=False)
    assert_bev_close(out.cpu().numpy(), ora["bev"])


def test_degenerate_all_points_masked_and_single_pillar():
    cfg, inp, g = load_lift_case("tiny_level")
    g2 = dict(g)
    g2["cam_t"] = g["cam_t"] + 1.0e4             # every point far outside the grid
    out, ranks = run_cuda(cfg, inp, g2, return_ranks=True)
    assert int((ranks >= 0).sum()) == 0 and float(out.abs().max()) == 0.0
    g3 = dict(g)
    g3["cam_M"] = np.zeros_like(g["cam_M"])      # every point collapses onto the camera centre: one pillar
    g3["ego_R"] = np.zeros_like(g["ego_R"]); g3["ego_t"] = np.zeros_like(g["ego_t"])
    out, ranks = run_cuda(cfg, inp, g3, return_ranks=True)
    ora = run_oracle(cfg, inp, g3)
    assert np.array_equal(ranks.cpu().numpy(), ora["rank"])
    assert_bev_close(out.cpu().numpy(), ora["bev"])


@pytest.mark.parametrize("seed", [5, 6])
def test_random_calibration_boundaries(seed):
    """Random (non-level) camera poses put many points on or near cell boundaries and in the (-1,0) truncation
    band; ranks must still be bit-exact with the oracle (which is pinned to the reference)."""
    cfg = syn.CONFIGS["carla_res"]
    inp = syn.lift_inputs(cfg, 2, seed=seed, random_pose=True)
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    g = dict(cam_M=cam_M.numpy(), cam_t=cam_t.numpy(), ego_R=ego_R.numpy(), ego_t=ego_t.numpy(), xs=xs.numpy(),
             ys=ys.numpy(), ds=ds.numpy(), bev_offset=G.bev_offset(start, res).numpy(), bev_resolution=res.numpy(),
             bev_dimension=dim.numpy())
    out, ranks = run_cuda(cfg, inp, g, return_ranks=True)
    ora = run_oracle(cfg, inp, g)
    assert np.array_equal(ranks.cpu().numpy(), ora["rank"])
    assert_bev_close(out.cpu().numpy(), ora["bev"])


def test_full_size_properties_batch4():
    """BASELINE perceive size, batch 4: size-independent properties (linearity in the features, mass conservation,
    batch independence) — the oracle itself only runs batch 1 in the golden test above."""
    cfg = syn.CONFIGS["perceive"]
    inp = syn.lift_inputs(cfg, 4, seed=2)
    dev = torch.device("cuda:0")
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    off = G.bev_offset(start, res)
    args = (cam_M, cam_t, ego_R, ego_t, xs, ys, ds, off, res, dim, cfg.discount)
    feat, dl = inp["feat"].to(dev), inp["depth_logits"].to(dev)
    out, ranks = ops.lift_splat(feat, dl, *args, return_ranks=True)
    out2 = ops.lift_splat(feat * 2.0, dl, *args)
    assert torch.allclose(out2, out * 2.0, rtol=1e-5, atol=1e-5)          # linear in the context features
    # mass conservation for frame 0 (no discount history): sum over cells == sum over kept points of p*f
    prob = dl.softmax(dim=3)
    keep = (ranks >= 0).float()
    mass = torch.einsum("bndhw,bnchw->bc", (prob[:, 0] * keep[:, 0]).double(), feat[:, 0].double())
    assert torch.allclose(out[:, 0].double().sum(dim=(-1, -2)), mass, rtol=1e-4)
    # each sample only depends on its own inputs
    out_b2 = ops.lift_splat(feat[2:3], dl[2:3], *(a[2:3] if torch.is_tensor(a) and a.dim() > 1 and a.shape[0] == 4 else a
                                                 for a in args))
    assert torch.allclose(out_b2[0], out[2], rtol=1e-5, atol=1e-5)


def test_workspace_is_left_clean_and_reusable():
    """finalize re-zeroes exactly what the scatter wrote: the workspace is all-zero after a call, and a second
    call on the same workspace (different inputs in between) reproduces the first result."""
    cfg, inp, g = load_lift_case("plumbing")
    ws = ops.Workspace()
    a = run_cuda(cfg, inp, g, workspace=ws).clone()
    torch.cuda.synchronize()
    assert int(ws.buf.count_nonzero()) == 0
    inp2 = dict(inp); inp2["feat"] = inp["feat"] * 3.0
    run_cuda(cfg, inp2, g, workspace=ws)
    b = run_cuda(cfg, inp, g, workspace=ws)
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-6)
    assert int(ws.buf.count_nonzero()) == 0


def test_workspace_clean_after_pool_sum_call_of_another_shape():
    """Regression: a call that emits pool sums must leave the shared workspace all-zero too (its per-CTA partials
    live in the workspace), otherwise a later call with a different shape would scatter into dirty memory."""
    ws = ops.Workspace()
    cfg, inp, g = load_lift_case("plumbing")
    run_cuda(cfg, inp, g, workspace=ws, pool_sum=True)
    torch.cuda.synchronize()
    assert int(ws.buf.count_nonzero()) == 0
    cfg2, inp2, g2 = load_lift_case("tiny_randpose")
    out = run_cuda(cfg2, inp2, g2, workspace=ws)
    assert_bev_close(out.cpu().numpy(), run_oracle(cfg2, inp2, g2)["bev"])


def test_stress_like_shapes_c128_d96_s5():
    """BASELINE configs[4] in miniature: C=128 (two 64-channel chunks in the scatter, two channel groups in the
    finalize), D=96 depth bins, S=5 frames (four chained ego poses), ranks bit-exact and BEV within tolerance."""
    cfg = syn.LiftSplatConfig(x_bound=(-20.0, 20.0, 0.5), y_bound=(-20.0, 20.0, 0.5), d_bound=(2.0, 98.0, 1.0),
                              final_dim=(64, 96), out_channels=128, n_cameras=3, receptive_field=5)
    inp = syn.lift_inputs(cfg, 2, seed=9, random_pose=True)
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    g = dict(cam_M=cam_M.numpy(), cam_t=cam_t.numpy(), ego_R=ego_R.numpy(), ego_t=ego_t.numpy(), xs=xs.numpy(),
             ys=ys.numpy(), ds=ds.numpy(), bev_offset=G.bev_offset(start, res).numpy(), bev_resolution=res.numpy(),
             bev_dimension=dim.numpy())
    out, ranks, psum = run_cuda(cfg, inp, g, return_ranks=True, pool_sum=True)
    ora = run_oracle(cfg, inp, g)
    assert np.array_equal(ranks.cpu().numpy(), ora["rank"])
    assert_bev_close(out.cpu().numpy(), ora["bev"])
    tot = ora["bev"].sum(axis=(-1, -2))
    assert np.allclose(psum.cpu().numpy(), tot, rtol=1e-4, atol=1e-4 * np.abs(tot).max())


def test_frame_sharded_raw_splats_plus_discount_equal_fused_path():
    """Frame-sharded mode on one GPU: two 'ranks' splat disjoint flat-frame ranges raw, the concatenation goes through
    stp3_bev_discount, and the bf16 hi/lo planes match the fused call's (same kernels; only atomic order differs)."""
    from stp3_b200 import parallel
    cfg, inp, g = load_lift_case("tiny_randpose")
    dev = torch.device("cuda:0")
    t = lambda a: torch.as_tensor(a).to(dev)
    args = (inp["feat"].to(dev), inp["depth_logits"].to(dev), t(g["cam_M"]), t(g["cam_t"]), t(g["ego_R"]), t(g["ego_t"]),
            t(g["xs"]), t(g["ys"]), t(g["ds"]), g["bev_offset"], g["bev_resolution"], g["bev_dimension"])
    B, S = inp["feat"].shape[:2]
    X, Y = int(g["bev_dimension"][0]), int(g["bev_dimension"][1])
    C = inp["feat"].shape[3]
    parts = []
    for r in range(2):
        f0, fc = parallel.shard_batch(B * S, r, 2)
        parts.append(ops.lift_splat_frames(*args, f0, fc))
    raw = torch.cat(parts).view(B, S, X, Y, C)
    ref = ops.lift_splat(*args, cfg.discount, out_channels_last=True)          # fused: fp32 channels-last
    rec = raw.clone()
    for s in range(1, S):
        rec[:, s] = rec[:, s - 1] * cfg.discount + raw[:, s]
    assert torch.allclose(rec, ref, rtol=1e-5, atol=1e-6 * float(ref.abs().max()))
    # C = 5 is not a multiple of 8: pad channels for the hi/lo kernel
    rawp = torch.zeros(B, S, X, Y, 8, device=dev); rawp[..., :C] = raw
    planes = ops.bev_discount(rawp, cfg.discount)
    got = (planes[0].float() + planes[1].float())[..., :C]
    assert (got - ref).abs().max() <= 2e-5 * ref.abs().max()


def test_frame_sharded_peer_stores_land_in_their_slots():
    """The all-gather fused into the finalize epilogue (peer_ptrs), with this device's own buffer as the only peer: the
    frames f_begin + [0, f_count) of each of two 'ranks' land in their slots and equal the raw splats of the same range."""
    from stp3_b200 import parallel
    dev = torch.device("cuda:0")
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
    inp = syn.lift_inputs(lcfg, 2, seed=7, random_pose=True)
    mats = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    res, start, dim = G.calculate_birds_eye_view_parameters(lcfg.x_bound, lcfg.y_bound, lcfg.z_bound)
    args = (inp["feat"].to(dev), inp["depth_logits"].to(dev), *mats,
            *G.frustum_axes(lcfg.final_dim, lcfg.downsample, lcfg.d_bound), G.bev_offset(start, res), res, dim)
    B, S, C = inp["feat"].shape[0], inp["feat"].shape[1], inp["feat"].shape[3]
    gathered = torch.full((B * S, int(dim[0]), int(dim[1]), C), float("nan"), device=dev)
    for r in range(2):
        f0, fc = parallel.shard_batch(B * S, r, 2)
        assert ops.lift_splat_frames(*args, f0, fc, peer_ptrs=[gathered.data_ptr()]) is None
        raw = ops.lift_splat_frames(*args, f0, fc)
        assert torch.allclose(gathered[f0:f0 + fc], raw, rtol=1e-5, atol=1e-6 * float(raw.abs().max()))
    assert not gathered.isnan().any()
