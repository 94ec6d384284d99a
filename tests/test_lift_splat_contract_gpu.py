"""GPU: the lift-splat forward on every kernel path stp3_lift_splat_plan can pick (the cases of
tests/lift_contract_cases.py), its backward on the shapes that stress the gradient kernel, and stp3_bev_discount, all
against float64 / bitwise host references.

Checked per forward case:
  - the plan the case is pinned to, and on the GPU no silent fall-back (scatter == tma_rules);
  - voxel ranks bit-exact against the oracle (oracle/lift_splat_oracle.py);
  - the BEV within the bars of test_lift_splat_gpu.assert_bev_close (2e-5 of max, 1e-3 relative above 1e-3 of max,
    exact zeros stay zero); the bf16 hi/lo planes as hi + lo, with a further 2^-17 |value| per element for the split;
  - pool sums within rtol 1e-4; every output element written (outputs pre-filled with NaN);
  - one workspace shared by the whole matrix, all-zero after every call;
  - TMA cases once more with feat at a 4-byte offset, which forces the generic kernel on the same inputs.
The last test asserts that the run reached every path of lift_contract_cases.PATHS."""
import os
import time

import numpy as np
import pytest
import torch

from oracle import lift_splat_oracle as O
from stp3_b200 import ops
from stp3_b200.utils import geometry as G
from stp3_b200.utils import synthetic as syn
from tests.lift_contract_cases import CASES, PATHS, XB2, YB2, path_labels

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NO_TMA = bool(int(os.environ.get("STP3_LIFT_NO_TMA", "0") or "0"))
ABS_BAR, REL_BAR = 2e-5, 1e-3      # of max |oracle|; relative above 1e-3 of max (test_lift_splat_gpu.assert_bev_close)
SPLIT = 2.0 ** -17                 # hi + lo is within 2^-18 |v| of the kernel's fp32 v (test_conv_contract_gpu.py)
GRAD_BAR = 1e-5                    # of max |oracle| (test_lift_splat_bwd_gpu.py)
WS = ops.Workspace()               # one workspace for every forward call of the module
REACHED = {}                       # case name -> path labels of the plans that ran


def geometry(cfg, inp):
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    return cam_M, cam_t, ego_R, ego_t, xs, ys, ds, G.bev_offset(start, res), res, dim


def oracle(inp, geo, discount, use_depth):
    a = [t.numpy() for t in geo]
    t0 = time.perf_counter()
    ora = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), *a, discount, use_depth_distribution=use_depth)
    return ora, time.perf_counter() - t0


def at_offset4(t):
    """t's values in a tensor whose storage starts 4 bytes past a 256-byte aligned allocation"""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    buf[1:].copy_(t.reshape(-1))
    return buf[1:].view(t.shape)


def bev_check(got, ref, split=0.0):
    """(error beyond the split allowance, of max |ref|; worst relative error above 1e-3 of max) after asserting the
    bars, that nothing is NaN and that exact zeros stay exact"""
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements never written"
    scale = np.abs(ref).max()
    assert scale > 0
    diff = np.maximum(np.abs(got - ref) - split * np.abs(ref), 0.0)
    big = np.abs(ref) > 1e-3 * scale
    err, rel = diff.max() / scale, (diff[big] / np.abs(ref[big])).max()
    assert err <= ABS_BAR and rel <= REL_BAR, (err, rel)
    assert not np.any(got[ref == 0] != 0), "an empty pillar is not exactly zero"
    return err, rel


def pillars_per_pair(ranks):
    """distinct pillars of every (sample, frame, camera, depth bin, image column) pair: ranks (B,S,N,D,Hf,Wf)"""
    r = np.sort(ranks, axis=4)
    new = r >= 0
    new[..., 1:, :] &= r[..., 1:, :] != r[..., :-1, :]
    return new.sum(axis=4)


def run_forward(case, feat, depth, geo, discount):
    """One call of the case into NaN-filled outputs; returns (B,S,C,X,Y) or (f_count,C,X,Y) float64, ranks, pool sums"""
    B, S, C = case.B, case.S, case.C
    X, Y = int(geo[-1][0]), int(geo[-1][1])
    kw = dict(feat_channels_last=case.nhwc, use_depth_distribution=case.use_depth)
    nan = float("nan")
    if case.frames:
        f0, fc = case.frames
        if case.n_peers:
            bufs = [torch.full((B * S, X, Y, C), nan, device=DEV) for _ in range(case.n_peers)]
            assert ops.lift_splat_frames(feat, depth, *geo, f0, fc, workspace=WS, peer_ptrs=[b.data_ptr() for b in bufs],
                                         **kw) is None
            torch.cuda.synchronize()
            for b in bufs:       # every slot outside the frame range is left alone, the two buffers are equal
                assert b[:f0].isnan().all() and b[f0 + fc:].isnan().all()
                assert torch.equal(b[f0:f0 + fc], bufs[0][f0:f0 + fc])
            out = bufs[0][f0:f0 + fc]
        else:
            desc, f, d = ops._lift_desc(feat, depth, *geo, 0.0, case.nhwc, case.use_depth, f0, fc)
            out = torch.full((fc, X, Y, C), nan, device=DEV)
            ops._lift_fwd(desc, f, d, WS, out, 1)
        return out.permute(0, 3, 1, 2).double().cpu().numpy(), None, None
    if case.out_layout == 2:
        kw["out_hilo"] = torch.full((2, B, S, X, Y, C), nan, dtype=torch.bfloat16, device=DEV)
    else:
        shape = (B, S, X, Y, C) if case.out_layout == 1 else (B, S, C, X, Y)
        kw["out"] = torch.full(shape, nan, device=DEV)
    res = ops.lift_splat(feat, depth, *geo, discount, out_channels_last=case.out_layout == 1, return_ranks=True,
                         pool_sum=case.pool_sum, workspace=WS, **kw)
    out, ranks = res[0], res[1]
    if case.out_layout == 2:
        out = out[0].double() + out[1].double()
    if case.out_layout != 0:
        out = out.permute(0, 1, 4, 2, 3)
    psum = res[2].double().cpu().numpy() if case.pool_sum else None
    return out.double().cpu().numpy(), ranks.cpu().numpy(), psum


def check_plan(case, plan):
    if NO_TMA:
        assert plan["tma_rules"] == 0 and plan["scatter"] == 0
        return
    assert {k: plan[k] for k in case.plan} == case.plan, (plan, case.plan)
    assert plan["scatter"] == plan["tma_rules"], "the TMA kernel is admissible but the tensor maps were not encoded"


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_forward_case_against_fp64(case):
    cfg = case.config()
    inp = syn.lift_inputs(cfg, case.B, seed=case.seed, random_pose=case.random_pose)
    geo = geometry(cfg, inp)
    discount = 0.0 if case.frames else cfg.discount
    ora, t_ora = oracle(inp, geo, discount, case.use_depth)
    ref = ora["bev"]
    if case.frames:
        f0, fc = case.frames
        ref = ref.reshape((-1,) + ref.shape[2:])[f0:f0 + fc]
    feat = inp["feat"].to(DEV)
    if case.nhwc:
        feat = feat.permute(0, 1, 2, 4, 5, 3).contiguous()
    depth = inp["depth_logits"].to(DEV)
    f0, fc = case.frames or (0, 0)
    pkw = dict(feat_channels_last=case.nhwc, use_depth_distribution=case.use_depth, f_begin=f0, f_count=fc,
               n_peers=case.n_peers, out_channels_last=case.out_layout == 1)
    if case.out_layout == 2:
        pkw["out_hilo"] = torch.empty(0)
    plan = ops.lift_splat_plan(feat, depth, *geo, discount, **pkw)
    check_plan(case, plan)
    REACHED[case.name] = path_labels(case, plan) if not NO_TMA else set()

    variants = [("aligned", feat, plan)]
    if plan["tma_rules"]:
        feat4 = at_offset4(feat)
        plan4 = ops.lift_splat_plan(feat4, depth, *geo, discount, **pkw)
        assert plan4["tma_rules"] == 0 and plan4["scatter"] == 0
        variants.append(("feat+4B", feat4, plan4))
    split = SPLIT if case.out_layout == 2 else 0.0
    line = []
    for tag, f, p in variants:
        got, ranks, psum = run_forward(case, f, depth, geo, discount)
        torch.cuda.synchronize()
        assert int(WS.buf.count_nonzero()) == 0, f"{tag}: the call left the workspace dirty"
        if ranks is not None:
            bad = int((ranks != ora["rank"]).sum())
            assert bad == 0, f"{tag}: {bad} voxel ranks differ from the oracle"
        err, rel = bev_check(got, ref, split)
        if case.pool_sum:
            tot = ref.sum(axis=(-1, -2))
            assert np.allclose(psum, tot, rtol=1e-4, atol=1e-4 * np.abs(tot).max()), f"{tag}: pool sums"
        line.append(f"{tag} {'TMA' if p['scatter'] else 'generic TW%d' % p['scatter_tw']}: err {err:.1e} rel {rel:.1e}")
    D = case.dims()["D"]
    if plan["tma_rules"] and D % 16:      # the partial last m-tile holds points that land in the grid
        assert (ora["rank"][:, :, :, D - D % 16:] >= 0).any()
    if case.leftovers:
        n = pillars_per_pair(ora["rank"])
        assert ((n >= 2) & (n <= 4)).any() and (n > 4).any(), np.bincount(n.reshape(-1))
        line.append(f"pairs over 2-4 pillars {int(((n >= 2) & (n <= 4)).sum())}, over >4 {int((n > 4).sum())}")
    d = case.dims()
    print(f"\n{case.name}: D={d['D']} Hf={d['Hf']} Wf={d['Wf']} C={case.C} S={case.S} plan={plan} | " + " | ".join(line)
          + f" | oracle {t_ora:.2f} s")


def test_every_path_is_reached():
    if NO_TMA:
        pytest.skip("STP3_LIFT_NO_TMA turns the TMA scatter off (read once per process)")
    missing = [c.name for c in CASES if c.name not in REACHED]
    assert not missing, f"cases not run: {missing}"
    reached = set().union(*REACHED.values())
    print("\n" + "\n".join(f"  {p:<42s} {sorted(n for n, r in REACHED.items() if p in r)}" for p in sorted(PATHS)))
    assert PATHS <= reached, PATHS - reached


# ------------------------------------------------------------------------------------------------ stp3_bev_discount
def bf16_bits(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy()


def test_bev_discount_is_the_fp32_recurrence_bit_for_bit():
    """out[t] = fp32(fp32(out[t-1] * discount) + raw[t]); hi = bf16_rn(out), lo = bf16_rn(out - hi)"""
    g = torch.Generator().manual_seed(11)
    for S in range(1, 9):
        for C in (8, 16, 128):
            raw = (torch.randn(2, S, 5, 7, C, generator=g) * torch.exp2(torch.randint(-8, 8, (2, S, 5, 7, C), generator=g)))
            raw[:, :, 1] = 0.0                                          # an empty row of cells
            for disc in (0.0, 0.5, 1.0):
                planes = ops.bev_discount(raw.to(DEV), disc)
                hi, lo = planes[0].view(torch.int16).cpu().numpy(), planes[1].view(torch.int16).cpu().numpy()
                r = raw.numpy()
                acc = np.zeros(r[:, 0].shape, np.float32)
                for t in range(S):
                    acc = (acc * np.float32(disc)).astype(np.float32) + r[:, t]
                    h = bf16_bits(acc)
                    h_f = torch.from_numpy(h).view(torch.bfloat16).float().numpy()
                    assert np.array_equal(hi[:, t], h), (S, C, disc, t)
                    assert np.array_equal(lo[:, t], bf16_bits(acc - h_f)), (S, C, disc, t)


# ------------------------------------------------------------------------------------------------ backward
BWD_CASES = [
    # name, d_bound, final_dim, C, S, N, use_depth, xb, yb
    ("bwd_c5_d41_hf7", (2.0, 10.2, 0.2), (56, 80), 5, 2, 2, True, (-11.25, 11.25, 0.5), (-9.5, 9.5, 0.5)),
    ("bwd_c96_d1_hf1", (2.0, 3.0, 1.0), (8, 48), 96, 1, 3, True, (-11.25, 11.25, 0.5), (-9.5, 9.5, 0.5)),
    ("bwd_c128_d41_hf40", (2.0, 10.2, 0.2), (320, 48), 128, 1, 1, True, (-11.25, 11.25, 0.5), (-9.5, 9.5, 0.5)),
    ("bwd_c192_hf7_s8_nodepth", (2.0, 18.0, 1.0), (56, 80), 192, 8, 1, False, (-11.25, 11.25, 0.5), (-9.5, 9.5, 0.5)),
    ("bwd_c64_d41_hf28_s8", (2.0, 10.2, 0.2), (224, 48), 64, 8, 1, True, XB2, YB2),
]


@pytest.mark.parametrize("name,d_bound,final_dim,C,S,N,use_depth,xb,yb", BWD_CASES, ids=[c[0] for c in BWD_CASES])
def test_backward_case_against_fp64(name, d_bound, final_dim, C, S, N, use_depth, xb, yb):
    cfg = syn.LiftSplatConfig(x_bound=xb, y_bound=yb, d_bound=d_bound, final_dim=final_dim, out_channels=C,
                              n_cameras=N, receptive_field=S)
    inp = syn.lift_inputs(cfg, 1, seed=4, random_pose=True)
    geo = geometry(cfg, inp)
    ora, _ = oracle(inp, geo, cfg.discount, use_depth)
    n = pillars_per_pair(ora["rank"])
    X, Y = int(geo[-1][0]), int(geo[-1][1])
    W = torch.randn(1, S, C, X, Y, generator=torch.Generator().manual_seed(2))
    t0 = time.perf_counter()
    ogf, ogd = O.lift_splat_backward(W.numpy(), inp["feat"].numpy(), inp["depth_logits"].numpy(), ora["rank"],
                                     cfg.discount, use_depth_distribution=use_depth)
    t_ora = time.perf_counter() - t0
    feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)
    runs = [ops.lift_splat_backward(W.to(DEV), feat, depth, *geo, cfg.discount, use_depth_distribution=use_depth)
            for _ in range(2)]
    torch.cuda.synchronize()
    (gf, gd), (gf2, gd2) = runs
    assert torch.equal(gf, gf2), "two backward calls differ"
    gf = gf.double().cpu().numpy()
    e_f = np.abs(gf - ogf).max() / np.abs(ogf).max()
    assert e_f <= GRAD_BAR, e_f
    assert not np.any(gf[ogf == 0] != 0), "grad_feat not exactly zero where every point of a pixel is masked"
    msg = f"grad_feat {e_f:.1e}"
    if use_depth:
        assert torch.equal(gd, gd2), "two backward calls differ"
        gd = gd.double().cpu().numpy()
        if ogd.shape[3] == 1:     # one depth bin: the softmax is constant, its gradient exactly zero
            assert not np.any(ogd != 0) and not np.any(gd != 0)
            msg += ", grad_depth exactly 0"
        else:
            e_d = np.abs(gd - ogd).max() / np.abs(ogd).max()
            assert e_d <= GRAD_BAR, e_d
            assert not np.any(gd[ogd == 0] != 0), "grad_depth not exactly zero where every point of a pixel is masked"
            msg += f", grad_depth {e_d:.1e}"
    else:
        assert gd is None
    print(f"\n{name}: {msg}; masked points {int((ora['rank'] < 0).sum())}, pairs over >1 pillar {int((n > 1).sum())}, "
          f"over >4 {int((n > 4).sum())} | oracle {t_ora:.2f} s")
