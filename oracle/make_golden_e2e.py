"""Generates tests/golden/e2e_perceive_*.npz: the UNMODIFIED reference (imported from the reference checkout through
oracle/ref_loader.py) run END TO END at the headline size -- lift-splat -> ego-motion concat -> TemporalModel(70, 3,
(200, 200)) -> Decoder (perceive gates) on ONE perceive-config sample (6 cameras x 3 frames, 200x200x64 BEV; ASPP
dilations 12/24/36 all live) -- next to the fp64 oracle on the same inputs.  Test infrastructure; run by hand in the
build container (about ten minutes on 8 cores):  python -m oracle.make_golden_e2e

The weights are the ones bench.py's model carries (synthetic.init_exact(STP3, seed=0): keyed by the state-dict names
of the whole model), loaded into the reference modules with strict=True; the inputs are synthetic.lift_inputs(perceive,
batch 1, seed) -- machine-independent -- so the GPU tests and bench.py regenerate them instead of shipping 43 MB.

Stored per case (level rig = SURVEY.md §8d's; tilted rig = every camera 1 degree off level): SHA-256 of the inputs and
of the reference's voxel ranks, and for the BEV features, the temporal model's output and every head's logits a
12k-entry random sample (int32 index, reference fp32 value, oracle fp64 value) plus max |value| (the normaliser of the
"relative to max" error the tests use).
"""
import copy
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.make_golden import run_reference, sha, OUT  # noqa: E402
from oracle.make_golden_dense import GATES_PERCEIVE  # noqa: E402
from oracle import lift_splat_oracle as O  # noqa: E402
from oracle import torch_dense as TD  # noqa: E402
from stp3_b200.utils import geometry as G  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402

CASES = [("level", 0, 0.0), ("tilted", 0, 1.0)]          # name, sample seed, tilt [deg]
N_SAMPLE = 12_000      # keeps each fixture below 1 MB


def shifted_ego(ego):
    return torch.cat([torch.zeros_like(ego[:, :1]), ego[:, :-1]], 1)


def sample_of(t_ref, t_ora, gen):
    flat_r, flat_o = t_ref.reshape(-1), t_ora.reshape(-1)
    idx = torch.randint(0, flat_r.numel(), (N_SAMPLE,), generator=gen)
    return {"index": idx.numpy().astype(np.int32), "ref": flat_r[idx].float().numpy(), "oracle": flat_o[idx].double().numpy(),
            "max": np.float64(flat_o.abs().max().item())}


def main():
    import bench
    ref = load_reference()
    cfg = syn.CONFIGS["perceive"]
    only = set(sys.argv[1:])
    with torch.no_grad():
        model = bench.build_model(lcfg=cfg)                      # drop-in module tree on the CPU: weights only
        X, Y = cfg.bev_xy
        ref_tm = ref.temporal_model.TemporalModel(70, 3, (X, Y), start_out_channels=64).eval()
        ref_tm.load_state_dict(model.temporal_model.state_dict(), strict=True)
        ref_dec = ref.decoder.Decoder(64, 2, 3, 2, GATES_PERCEIVE).eval()
        ref_dec.load_state_dict(model.decoder.state_dict(), strict=True)
        m64 = copy.deepcopy(model).double()
        for name, seed, tilt in CASES:
            if only and name not in only:
                continue
            t0 = time.time()
            inp = syn.lift_inputs(cfg, 1, seed=seed, tilt_deg=tilt)
            fake, geom, rank, bev = run_reference(ref, cfg, inp)
            ego = shifted_ego(inp["future_egomotion"])
            x = torch.cat([bev, ego.view(1, -1, 6, 1, 1).expand(1, ego.shape[1], 6, X, Y)], dim=2)
            states = ref_tm(x)
            out = ref_dec(states)
            t1 = time.time()
            # fp64 oracle on the same inputs
            cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
            xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
            res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
            ora = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), cam_M.numpy(), cam_t.numpy(),
                               ego_R.numpy(), ego_t.numpy(), xs.numpy(), ys.numpy(), ds.numpy(),
                               G.bev_offset(start, res).numpy(), res.numpy(), dim.numpy(), cfg.discount)
            assert np.array_equal(ora["rank"].reshape(-1), rank.numpy().reshape(-1)), "oracle ranks != reference ranks"
            bev64 = torch.from_numpy(ora["bev"])
            x64 = torch.cat([bev64, ego.double().view(1, -1, 6, 1, 1).expand(1, ego.shape[1], 6, X, Y)], dim=2)
            states64 = TD.temporal_model(x64, m64.temporal_model)
            out64 = TD.decoder(states64, m64.decoder)
            t2 = time.time()
            gen = torch.Generator().manual_seed(4321)
            rec = dict(config="perceive", seed=seed, tilt_deg=tilt, weights_seed=0,
                       feat_sha=sha(inp["feat"].numpy()), depth_sha=sha(inp["depth_logits"].numpy()),
                       rank_sha=sha(rank.numpy()), n_kept=int((rank >= 0).sum()),
                       intrinsics=inp["intrinsics"].numpy(), extrinsics=inp["extrinsics"].numpy(),
                       future_egomotion=inp["future_egomotion"].numpy(),
                       cam_M=cam_M.numpy(), cam_t=cam_t.numpy(), ego_R=ego_R.numpy(), ego_t=ego_t.numpy())
            for key, (r32, r64) in {"bev": (bev, bev64), "states": (states, states64),
                                    "segmentation": (out["segmentation"], out64["segmentation"]),
                                    "pedestrian": (out["pedestrian"], out64["pedestrian"]),
                                    "hdmap": (out["hdmap"], out64["hdmap"])}.items():
                s = sample_of(r32, r64, gen)
                dev = np.abs(s["ref"].astype(np.float64) - s["oracle"]).max() / s["max"]
                print(f"  {key:13s} shape {tuple(r32.shape)}  max|.| {s['max']:.4g}  reference fp32 vs oracle fp64: {dev:.2e} of max")
                for k2, v in s.items():
                    rec[f"{key}_{k2}"] = v
            path = os.path.join(OUT, f"e2e_perceive_{name}.npz")
            np.savez_compressed(path, **rec)
            print(f"{name}: reference {t1 - t0:.0f} s, oracle {t2 - t1:.0f} s -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
