"""GPU: the deterministic mode (torch.use_deterministic_algorithms; DESIGN.md §3.14).

  - every lift-splat contract case (tests/lift_contract_cases.py: both scatter kernels, NCHW / NHWC, C = 64 and more,
    with and without the depth distribution, every output layout with pool sums, frame ranges and peer stores) run
    twice under the flag into NaN-filled outputs with one reused workspace: outputs, ranks and pool sums bitwise equal,
    the workspace all-zero afterwards, ranks bit-exact and the BEV within the fp64-oracle bars of the default path;
  - the generic kernel without depth distribution equals a host model of the fixed-point scheme bit for bit;
  - a sample's BEV does not depend on the batch it sits in, nor a frame's on the frame range of the call;
  - a +inf depth logit poisons exactly the pillars its pixel's points reach, in every channel, from that frame on; a
    NaN feature poisons those and at most other pillars of its image column (0 * NaN in the column's products);
  - default and fixed-point calls interleaved on one workspace;
  - stp3_spatial_sum_det: within the fp64 bar and bitwise repeatable;
  - a small native-trunk STP3: eval forwards, CUDA graphs against eager, two train_heads() steps in fp32 and under fp16
    autocast with GradScaler, and two processes, all bitwise equal;
  - a graph captured without the flag keeps its workspace when an eager call under the flag replaces the model's;
  - on two GPUs, frames gathered by NCCL and by peer stores equal the unsharded splat bit for bit."""
import contextlib
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from stp3_b200 import dense, ops
from stp3_b200.utils import synthetic as syn
from tests import test_deterministic_cpu as M
from tests.lift_contract_cases import CASES, Case
from tests.test_lift_splat_contract_gpu import bev_check, geometry, oracle, run_forward, SPLIT, WS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def case_inputs(case, B=None, seed=None):
    cfg = case.config()
    inp = syn.lift_inputs(cfg, B or case.B, seed=case.seed if seed is None else seed, random_pose=case.random_pose)
    geo = geometry(cfg, inp)
    feat = inp["feat"].to(DEV)
    if case.nhwc:
        feat = feat.permute(0, 1, 2, 4, 5, 3).contiguous()
    return cfg, inp, geo, feat, inp["depth_logits"].to(DEV)


# ------------------------------------------------------------------------------------------------ contract
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_fixed_point_case_repeatable_and_against_fp64(case):
    cfg, inp, geo, feat, depth = case_inputs(case)
    discount = 0.0 if case.frames else cfg.discount
    ora, _ = oracle(inp, geo, discount, case.use_depth)
    ref = ora["bev"]
    if case.frames:
        f0, fc = case.frames
        ref = ref.reshape((-1,) + ref.shape[2:])[f0:f0 + fc]
    runs = []
    with deterministic():
        for _ in range(2):
            runs.append(run_forward(case, feat, depth, geo, discount))
            torch.cuda.synchronize()
            assert int(WS.buf.count_nonzero()) == 0, "the call left the workspace dirty"
    (a, ra, pa), (b, rb, pb) = runs
    assert np.array_equal(a, b, equal_nan=True), "two fixed-point runs differ"
    if ra is not None:
        assert np.array_equal(ra, rb) and np.array_equal(ra, ora["rank"]), "voxel ranks"
    if case.pool_sum:
        assert np.array_equal(pa, pb), "pool sums differ between runs"
        tot = ref.sum(axis=(-1, -2))
        assert np.allclose(pa, tot, rtol=1e-4, atol=1e-4 * np.abs(tot).max()), "pool sums"
    err, rel = bev_check(a, ref, SPLIT if case.out_layout == 2 else 0.0)
    print(f"\n{case.name}: err {err:.1e} rel {rel:.1e} of the fp64 oracle")


# ------------------------------------------------------------------------------------------------ exact host model
EXACT = Case("det_exact_generic", (2.0, 18.0, 1.0), (64, 80), 33, 3, use_depth=False, out_layout=1)


def test_generic_kernel_without_depth_equals_the_host_model_bit_for_bit():
    """use_depth_distribution = 0: every probability is exactly 1, so each flushed partial is a plain fp32 add chain
    over the rows of an image column (one chain when all its points share a pillar, one per run of equal ranks
    otherwise), and the whole output follows from M.fixed_point_bev."""
    case = EXACT
    cfg, inp, geo, feat, depth = case_inputs(case)
    # one large feature per frame makes k_f small, so the grid is coarser than the partials' ulps and rounding (not
    # truncation) is what the bits show
    inp["feat"][:, :, 0, 0, 0, 0] = 2.0 ** 40
    feat = inp["feat"].to(DEV)
    plan = ops.lift_splat_plan(feat, depth, *geo, cfg.discount, use_depth_distribution=False, out_channels_last=True)
    assert plan["scatter"] == 0 and plan["tma_rules"] == 0
    with deterministic():
        out, ranks = ops.lift_splat(feat, depth, *geo, cfg.discount, use_depth_distribution=False,
                                    out_channels_last=True, return_ranks=True, workspace=WS)
    nx, ny = cfg.bev_xy
    want = M.fixed_point_bev(inp["feat"].numpy(), ranks.cpu().numpy(), nx * ny, np.float32(cfg.discount))
    got = out.cpu().numpy().reshape(want.shape)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
        f"{int((got.view(np.uint32) != want.view(np.uint32)).sum())} values differ from the host model"
    assert np.abs(want).max() > 0


# ------------------------------------------------------------------------------------------------ invariance
@pytest.mark.parametrize("name", ["tma_d41_hf7", "gen_c96"])
def test_a_sample_does_not_depend_on_its_batch(name):
    base = next(c for c in CASES if c.name == name)
    case = dataclasses.replace(base, B=3)
    cfg, inp, geo, feat, depth = case_inputs(case, B=3, seed=2)
    feat[0] *= 16            # the batch's largest features sit in another sample: a per-call scale would show
    one = [t[1:2] for t in geo[:4]]
    with deterministic():
        all3 = ops.lift_splat(feat, depth, *geo, cfg.discount, workspace=WS)
        solo = ops.lift_splat(feat[1:2].contiguous(), depth[1:2].contiguous(), *one, *geo[4:], cfg.discount,
                              workspace=WS)
    assert torch.equal(all3[1:2], solo), "sample 1 differs between a B = 3 and a B = 1 call"


def test_frame_ranges_give_the_same_frames():
    case = next(c for c in CASES if c.name == "frames_c64")
    cfg, inp, geo, feat, depth = case_inputs(case)
    n = case.B * case.S
    feat = feat.clone()
    feat[0, 0] *= 16         # frames of different magnitude: a per-call scale would make frames depend on the range
    with deterministic():
        whole = ops.lift_splat_frames(feat, depth, *geo, 0, n, workspace=WS)
        parts = [ops.lift_splat_frames(feat, depth, *geo, f0, fc, workspace=WS) for f0, fc in ((0, 1), (1, 3), (4, 2))]
    assert torch.equal(whole, torch.cat(parts)), "a frame's splat depends on the frame range of the call"


# ------------------------------------------------------------------------------------------------ non-finite values
@pytest.mark.parametrize("what", ["nan_feature", "inf_depth_logit"])
@pytest.mark.parametrize("name", ["tma_d41_hf7", "gen_c33_nchw"])
def test_non_finite_values_poison_their_pillars(what, name):
    case = next(c for c in CASES if c.name == name)
    cfg, inp, geo, feat, depth = case_inputs(case)
    with deterministic():
        clean, ranks = ops.lift_splat(feat, depth, *geo, cfg.discount, return_ranks=True, workspace=WS)
    ranks = ranks.cpu().numpy()
    b, t, n = 0, 0, case.N - 1
    hit = np.argwhere(ranks[b, t, n] >= 0)          # (d, h, w) of points inside the grid
    d, h, w = hit[len(hit) // 2]
    feat2, depth2 = feat.clone(), depth.clone()
    if what == "nan_feature":
        feat2[b, t, n, 3, h, w] = float("nan")
    else:
        depth2[b, t, n, d, h, w] = float("inf")
    with deterministic():
        out = ops.lift_splat(feat2, depth2, *geo, cfg.discount, workspace=WS)
        torch.cuda.synchronize()
    assert int(WS.buf.count_nonzero()) == 0
    nx, ny = cfg.bev_xy
    o = out.cpu().numpy().reshape(case.B, case.S, case.C, nx * ny)
    reached = np.unique(ranks[b, t, n, :, h, w][ranks[b, t, n, :, h, w] >= 0])
    assert len(reached)
    nanp = np.isnan(o)
    assert nanp[b, t:][:, :, reached].all(), "a reached pillar is not NaN in every channel from its frame on"
    any_nan = nanp.any(axis=2)
    assert (any_nan == nanp.all(axis=2)).all(), "a pillar is NaN in some channels only"
    assert not any_nan[:, :t].any() and not any_nan[1:].any(), "NaN outside the sample's later frames"
    if what == "inf_depth_logit":          # the pixel's points only
        expect = np.zeros(nx * ny, bool)
        expect[reached] = True
        assert (any_nan[b, t] == expect).all()
    else:                                  # 0 * NaN reaches the other pillars of the same image column at most
        col = np.unique(ranks[b, t, n, :, :, w][ranks[b, t, n, :, :, w] >= 0])
        assert set(np.flatnonzero(any_nan[b, t])) <= set(col)
    fin = ~any_nan
    c = clean.cpu().numpy().reshape(o.shape)
    assert np.isfinite(o.transpose(0, 1, 3, 2)[fin]).all()
    if what == "inf_depth_logit":          # other pillars keep their bits
        assert np.array_equal(o.transpose(0, 1, 3, 2)[fin], c.transpose(0, 1, 3, 2)[fin])


# ------------------------------------------------------------------------------------------------ mode switching
def test_default_and_fixed_point_calls_interleave_on_one_workspace():
    case = next(c for c in CASES if c.name == "tma_c192_nhwc_s5")
    cfg, inp, geo, feat, depth = case_inputs(case)
    kw = dict(feat_channels_last=True, out_channels_last=True, pool_sum=True)
    ws = ops.Workspace()
    with deterministic():
        ref_det = ops.lift_splat(feat, depth, *geo, cfg.discount, workspace=ops.Workspace(), **kw)
    ref = ops.lift_splat(feat, depth, *geo, cfg.discount, workspace=ops.Workspace(), **kw)
    for det in (False, True, True, False, True, False):
        with deterministic(det):
            got = ops.lift_splat(feat, depth, *geo, cfg.discount, workspace=ws, **kw)
        torch.cuda.synchronize()
        assert int(ws.buf.count_nonzero()) == 0
        if det:
            assert all(torch.equal(a, b) for a, b in zip(got, ref_det))
        else:
            scale = ref[0].abs().max()
            assert (got[0] - ref[0]).abs().max() <= 1e-5 * scale
            assert torch.allclose(got[1], ref[1], rtol=1e-4, atol=1e-4 * ref[1].abs().max().item())


# ------------------------------------------------------------------------------------------------ spatial sums
@pytest.mark.parametrize("n_img,H,W,C,cstride", [(6, 25, 40, 64, 64), (2, 50, 50, 70, 128), (3, 7, 9, 1000, 1024),
                                                 (65535, 1, 2, 4, 8), (4, 200, 200, 64, 64)])
def test_spatial_sum_det(n_img, H, W, C, cstride):
    g = torch.Generator().manual_seed(n_img + cstride)
    x = torch.zeros(n_img, H, W, cstride)
    x[..., :C] = torch.randn(n_img, H, W, C, generator=g) * 3 + 1
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    hl = dense.HL(hi.view(n_img, 1, H, W, cstride).to(DEV), lo.view(n_img, 1, H, W, cstride).to(DEV), C)
    with deterministic():
        a = dense.spatial_sum(hl)
        b = dense.spatial_sum(hl)
    assert torch.equal(a, b), "stp3_spatial_sum_det is not repeatable"
    v = (hi.double() + lo.double()).sum(dim=(1, 2))
    got = a.cpu().double()
    assert (got[:, C:] == 0).all(), "padding channels"
    bar = 2.0 ** -23 * v.abs() + 1e-12 * (hi.double() + lo.double()).abs().sum(dim=(1, 2))
    assert ((got - v).abs() <= bar).all(), (got - v).abs().max()
    default = dense.spatial_sum(hl).cpu().double()       # the atomic path agrees to its own bar
    assert ((default - v).abs() <= 1e-5 * v.abs().max()).all()


# ------------------------------------------------------------------------------------------------ whole model
def small_model():
    from tests.test_encoder_train_gpu import small_stp3
    torch.manual_seed(0)             # the native trunk keeps torch's default initialisation
    model, inp = small_stp3("native")
    return model, inp


def image_of(seed):
    from tests.test_encoder_train_gpu import LCFG
    g = torch.Generator().manual_seed(seed)
    return torch.randn((1, 3, 2, 3, *LCFG.final_dim), generator=g).to(DEV)


def outputs(out):
    return {k: v.detach().clone() for k, v in out.items() if torch.is_tensor(v)}


def bits_equal(a, b):
    """equal bit patterns (NaN included)"""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.is_floating_point():
        view = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
        return torch.equal(a.contiguous().view(view), b.contiguous().view(view))
    return torch.equal(a, b)


def assert_bitwise(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert bits_equal(a[k], b[k]), f"{what}: {k}"


def test_eval_forward_and_graphs_are_bitwise_equal(monkeypatch):
    from stp3_b200.models.stp3 import GraphedPerception
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    model, inp = small_model()
    model.eval()
    image = image_of(3)
    args = (inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    with deterministic(), torch.no_grad():
        e1 = outputs(model(image, *args))
        e2 = outputs(model(image, *args))
        assert_bitwise(e1, e2, "two eager forwards")
        g = GraphedPerception(model, 1, 2, entry="images")
        gi = outputs(g(image, None, *args))
        assert_bitwise({k: gi[k] for k in e1 if k in gi}, {k: e1[k] for k in e1 if k in gi}, "graph (images) vs eager")
        feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)
        el = outputs(model.forward_features(feat, depth, *args))
        gl = GraphedPerception(model, 1, 2, entry="lift")
        gg = outputs(gl(feat, depth, *args))
        assert_bitwise({k: gg[k] for k in el if k in gg}, {k: el[k] for k in el if k in gg}, "graph (lift) vs eager")


def train_two_steps(amp):
    from tests.test_encoder_train_gpu import loss_of
    results = []
    for _ in range(2):
        model, inp = small_model()
        model.eval()
        model.encoder.train_heads()
        model.temporal_model.train()
        model.decoder.train()
        opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
        scaler = torch.amp.GradScaler("cuda", init_scale=1.0) if amp else None
        image = image_of(5)
        torch.manual_seed(11)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
            loss = loss_of(out)
        (scaler.scale(loss) if amp else loss).backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        if amp:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        torch.cuda.synchronize()
        results.append((loss.detach().clone(), grads, {k: b.clone() for k, b in model.named_buffers()},
                        {k: p.detach().clone() for k, p in model.named_parameters()}))
    return results


@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "fp16_autocast"])
def test_train_heads_steps_are_bitwise_equal(amp, monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    with deterministic(warn_only=True):
        (l1, g1, b1, p1), (l2, g2, b2, p2) = train_two_steps(amp)
    assert torch.equal(l1, l2), (l1.item(), l2.item())
    assert g1.keys() == g2.keys() and len(g1) > 0
    for what, x, y in (("gradient", g1, g2), ("buffer", b1, b2), ("parameter", p1, p2)):
        for k in x:
            assert bits_equal(x[k], y[k]), f"{what} {k}"


PROBE = r"""
import hashlib, sys, torch
sys.path.insert(0, sys.argv[1])
from tests.test_encoder_train_gpu import small_stp3, LCFG
torch.use_deterministic_algorithms(True)
torch.manual_seed(0)
model, inp = small_stp3("native")
model.eval()
g = torch.Generator().manual_seed(3)
image = torch.randn((1, 3, 2, 3, *LCFG.final_dim), generator=g).to("cuda:0")
with torch.no_grad():
    out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
h = hashlib.sha256()
for k in sorted(out):
    if torch.is_tensor(out[k]):
        h.update(k.encode()); h.update(out[k].detach().float().cpu().numpy().tobytes())
print("DIGEST", h.hexdigest())
"""


def test_two_processes_give_the_same_digest():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env.pop("STP3_CONV_AUTOTUNE", None)
    digests = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", PROBE, ROOT], capture_output=True, text=True, env=env, cwd=ROOT,
                           timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        digests.append([l for l in r.stdout.splitlines() if l.startswith("DIGEST")][-1])
    assert digests[0] == digests[1], digests


# ------------------------------------------------------------------------------------------------ graphs and workspace
def test_graph_keeps_its_workspace_when_an_eager_call_under_the_flag_grows_it(monkeypatch):
    """A graph captured with the flag off splats into the model's workspace; an eager call under the flag needs the
    larger fixed-point workspace and replaces the model's buffer.  The graph keeps the buffer it captured: blocks
    allocated afterwards are left alone, and the replay still matches eager."""
    from stp3_b200.models.stp3 import GraphedPerception
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    model, inp = small_model()
    model.eval()
    feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)
    args = (inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    with torch.no_grad():
        g = GraphedPerception(model, 1, 2, entry="lift")
        old_ptr, old_bytes = model._ws.buf.data_ptr(), model._ws.buf.numel()     # no reference kept here
        with deterministic():
            model.forward_features(feat, depth, *args)
        assert model._ws.buf.data_ptr() != old_ptr and model._ws.buf.numel() > old_bytes
        assert any(t.data_ptr() == old_ptr for t in g._keepalive if torch.is_tensor(t))
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        junk = [torch.full((old_bytes // 4,), 7.0, device=DEV) for _ in range(4)]
        eager = outputs(model.forward_features(feat, depth, *args))
        got = outputs(g(feat, depth, *args))
        torch.cuda.synchronize()
    assert all(bool((j == 7.0).all()) for j in junk), "the replay wrote into memory it does not own"
    for k in ("segmentation", "pedestrian", "hdmap"):       # the default path sums with atomics: test_trunk_gpu's bar
        assert (got[k] - eager[k]).abs().max() <= 1e-4 * eager[k].abs().max(), k


# ------------------------------------------------------------------------------------------------ two GPUs
def _two_gpu_worker(rank, world, port, q):
    import torch.distributed as dist
    from stp3_b200 import parallel
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    torch.use_deterministic_algorithms(True)
    try:
        res = {}
        for name in ("frames_c64", "frames_peers_c32"):         # TMA and generic scatter
            case = next(c for c in CASES if c.name == name)
            cfg = case.config()
            inp = syn.lift_inputs(cfg, case.B, seed=case.seed, random_pose=case.random_pose)
            geo = geometry(cfg, inp)
            feat, depth = inp["feat"].to(dev), inp["depth_logits"].to(dev)
            n = case.B * case.S
            ws = ops.Workspace()
            full = ops.lift_splat_frames(feat, depth, *geo, 0, n, workspace=ws)
            f0, fc = parallel.shard_batch(n, rank, world)
            nccl = parallel.all_gather_frames(ops.lift_splat_frames(feat, depth, *geo, f0, fc, workspace=ws), n)
            pf = parallel.PeerFrameBuffer(n, *full.shape[1:], dev)
            pf.barrier()
            ops.lift_splat_frames(feat, depth, *geo, f0, fc, workspace=ws, peer_ptrs=pf.ptrs)
            pf.barrier()
            torch.cuda.synchronize()
            res[name] = (bool(torch.equal(nccl, full)), bool(torch.equal(pf.buf, full)))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_sharded_frames_equal_the_unsharded_splat_on_two_gpus():
    """Frames splatted on two ranks and gathered by NCCL or by the finalize's peer stores equal the unsharded
    fixed-point splat bit for bit (a frame's scale is its own)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_gpu_worker, args=(r, 2, 29653, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, r in res:
        for name, (nccl_eq, peer_eq) in r.items():
            assert nccl_eq, (rank, name, "nccl")
            assert peer_eq, (rank, name, "peer")
