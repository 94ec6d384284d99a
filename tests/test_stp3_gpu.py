"""GPU: the assembled drop-in STP3 (perception configuration) end to end against the composed oracle
(numpy lift-splat in fp64 -> torch fp64 TemporalModel -> torch fp64 Decoder) with identical weights and inputs."""
import copy

import numpy as np
import pytest
import torch

from oracle import lift_splat_oracle as O
from oracle import torch_dense as TD
from stp3_b200.config import get_cfg
from stp3_b200.models.stp3 import STP3
from stp3_b200.utils import geometry as G
from stp3_b200.utils import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class FakeTrunk(torch.nn.Module):
    """Stands in for the third-party EfficientNet trunk (absent from the image): deterministic endpoints."""

    def forward(self, x):
        m = x.shape[0]
        g = torch.Generator().manual_seed(3)
        h, w = x.shape[-2] // 8, x.shape[-1] // 8
        r3 = TD.exact_gauss((m, 56, h, w), g).to(x.device)
        r4 = TD.exact_gauss((m, 160, h // 2, w // 2), g).to(x.device)
        return r3, r4


def small_cfg(extra=None):
    d = {"LIFT": {"X_BOUND": [-8.0, 8.0, 0.5], "Y_BOUND": [-8.0, 8.0, 0.5], "D_BOUND": [2.0, 10.0, 1.0]},
         "IMAGE": {"FINAL_DIM": (32, 48)}}
    for k, v in (extra or {}).items():
        if isinstance(v, dict):
            d.setdefault(k, {}).update(v)
        else:
            d[k] = v
    return get_cfg(d)


@pytest.mark.parametrize("C,S", [(64, 3), (128, 5)])      # perceive shape; stress shape (BASELINE configs[4]: C=128, S=5)
def test_forward_features_matches_composed_oracle(C, S):
    cfg = small_cfg({"TIME_RECEPTIVE_FIELD": S, "MODEL": {"ENCODER": {"OUT_CHANNELS": C}}} if (C, S) != (64, 3) else None)
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=C, n_cameras=2, receptive_field=S)
    inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
    with torch.no_grad():
        model = TD.init_exact(STP3(cfg, backbone=FakeTrunk()), seed=7).eval()
        # init_exact also rewrote the geometry buffers: restore them
        model.frustum.copy_(model.create_frustum()); 
        res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
        ref_model = copy.deepcopy(model).double()
        model = model.to(DEV)
        out = model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                     inp["extrinsics"], inp["future_egomotion"])
        # ---- oracle
        cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        xs, ys, ds = G.frustum_axes(cfg.IMAGE.FINAL_DIM, 8, cfg.LIFT.D_BOUND)
        bev = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), cam_M.numpy(), cam_t.numpy(), ego_R.numpy(),
                           ego_t.numpy(), xs.numpy(), ys.numpy(), ds.numpy(), G.bev_offset(start, res).numpy(),
                           res.numpy(), dim.numpy(), cfg.LIFT.DISCOUNT)["bev"]
        x = torch.from_numpy(bev)                                            # (B,S,64,X,Y) fp64
        ego = inp["future_egomotion"].double()
        ego = torch.cat([torch.zeros_like(ego[:, :1]), ego[:, :-1]], 1)      # stp3.py:148-151
        x = torch.cat([x, ego.view(2, S, 6, 1, 1).expand(2, S, 6, *x.shape[-2:])], dim=2)
        states = TD.temporal_model(x, ref_model.temporal_model)
        ref = TD.decoder(states, ref_model.decoder)
    assert out["depth_prediction"].shape == inp["depth_logits"].shape and out["cam_front"] is None
    for k in ("segmentation", "pedestrian", "hdmap"):
        r = ref[k]
        err = (out[k].double().cpu() - r).abs().max().item()
        assert out[k].shape == r.shape
        assert err <= 1e-3 * r.abs().max().item(), (k, err, r.abs().max().item())      # north_star: logits within 1e-3
    for k in ("instance_center", "instance_offset", "instance_flow", "costvolume"):
        assert out[k] is None


def test_forward_from_images_runs_with_injected_trunk():
    cfg = small_cfg()
    with torch.no_grad():
        model = STP3(cfg, backbone=FakeTrunk()).eval().to(DEV)
        lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                                   final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
        inp = syn.lift_inputs(lcfg, 1, seed=5)
        image = torch.zeros(1, 3, 2, 3, 32, 48, device=DEV)
        out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        bev, depth, cam_front = model.calculate_birds_eye_view_features(image, inp["intrinsics"], inp["extrinsics"],
                                                                        inp["future_egomotion"])
    assert out["segmentation"].shape == (1, 3, 2, 32, 32) and out["hdmap"].shape == (1, 4, 32, 32)
    assert out["depth_prediction"].shape == (1, 3, 2, 8, 4, 6)
    assert bev.shape == (1, 3, 64, 32, 32) and depth.shape == (1, 3, 2, 8, 4, 6) and cam_front is None
    assert all(torch.isfinite(v).all() for v in out.values() if v is not None)


def test_cuda_graph_replay_equals_eager():
    """GraphedPerception (one CUDA graph per step) returns exactly what the eager launch sequence returns, also when
    it is replayed with new inputs (lift-splat workspace invariants hold across replays)."""
    from stp3_b200.models.stp3 import GraphedPerception
    cfg = small_cfg()
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
    with torch.no_grad():
        model = syn.init_exact(STP3(cfg, backbone=FakeTrunk()), seed=8).eval()
        model.frustum.copy_(model.create_frustum())
        res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
        model = model.to(DEV)
        g = GraphedPerception(model, 2, 2)
        for seed in (1, 2, 1):
            inp = syn.lift_inputs(lcfg, 2, seed=seed, random_pose=True)
            args = (inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"], inp["extrinsics"],
                    inp["future_egomotion"])
            eager = model.forward_features(*args)
            out = g(*args)
            torch.cuda.synchronize()
            for k in ("segmentation", "pedestrian", "hdmap"):
                # identical kernels and launch order; only the lift-splat's atomic summation order may differ
                assert (out[k] - eager[k]).abs().max() <= 1e-4 * eager[k].abs().max(), k


def test_pipelined_front_end_matches_eager():
    """PipelinedPerception (copies overlapped with graph replays, two slots) returns the eager results in order."""
    from stp3_b200.models.stp3 import PipelinedPerception
    cfg = small_cfg()
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
    with torch.no_grad():
        model = syn.init_exact(STP3(cfg, backbone=FakeTrunk()), seed=8).eval()
        model.frustum.copy_(model.create_frustum())
        res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
        model = model.to(DEV)
        pipe = PipelinedPerception(model, 2, 2)
        inputs = [syn.lift_inputs(lcfg, 2, seed=s, random_pose=True) for s in (1, 2, 3)]
        pinned = [{k: v.pin_memory() for k, v in i.items()} for i in inputs]
        got = []
        for k, h in enumerate(pinned):
            pipe.submit(h["feat"], h["depth_logits"], h["intrinsics"], h["extrinsics"], h["future_egomotion"])
            if k >= 1:
                got.append({key: t.clone() for key, t in pipe.collect().items()})
        got.append({key: t.clone() for key, t in pipe.collect().items()})
        for inp, out in zip(inputs, got):
            eager = model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                           inp["extrinsics"], inp["future_egomotion"])
            for key in ("segmentation", "pedestrian", "hdmap"):
                assert (out[key] - eager[key].cpu()).abs().max() <= 1e-4 * eager[key].abs().max(), key


def _sharded_worker(rank, world_size, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world_size, device_id=dev)
    try:
        cfg = small_cfg()
        lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                                   final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
        with torch.no_grad():
            model = syn.init_exact(STP3(cfg, backbone=FakeTrunk()), seed=8).eval()
            model.frustum.copy_(model.create_frustum())
            res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
            model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
            model = model.to(dev)
            inp = syn.lift_inputs(lcfg, 1, seed=3, random_pose=True)        # global batch 1 < 2 GPUs
            a = (inp["feat"].to(dev), inp["depth_logits"].to(dev), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
            full = model.forward_features(*a)
            err = 0.0
            for gather in ("nccl", "peer", "peer"):       # "peer": finalize epilogue stores into every rank's buffer (NVLink)
                sharded = model.forward_features_frame_sharded(*a, gather=gather)
                torch.cuda.synchronize()
                err = max([err] + [float((sharded[k] - full[k]).abs().max() / full[k].abs().max())
                                   for k in ("segmentation", "pedestrian", "hdmap")])
        q.put((rank, err))
    finally:
        dist.destroy_process_group()


def test_frame_sharded_forward_two_gpus_nccl():
    """North-star multi-GPU mode: batch 1 split by camera frame over 2 GPUs; the raw BEV frames are exchanged by one
    NCCL all-gather, or by the finalize kernel's own peer stores over NVLink (symmetric memory) -- both must reproduce the
    unsharded forward."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, 29641, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(err <= 1e-4 for _, err in res), res
