"""Generates tests/golden/lift_splat_*.npz by running the UNMODIFIED reference (imported from
the reference checkout through oracle/ref_loader.py) on seeded synthetic inputs, on the CPU of the build
container.  Test infrastructure; run by hand:  python -m oracle.make_golden [case ...]

The reference has no tests/fixtures of its own (SURVEY.md §4), so these files are what pins the
oracle (oracle/lift_splat_oracle.py) and, through it, the CUDA path.  What is stored:

  small cases  : every input + the reference's warped geometry, voxel ranks and pooled BEV (fp32)
  large cases  : host parameters, SHA-256 of the (machine-independent, integer-generated) inputs,
                 SHA-256 of the reference's rank array, per-(t,c) sums and a 40k-entry random sample of
                 the reference's BEV output (a full perceive output is 30 MB and does not belong in git)
"""
import hashlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference, make_fake_stp3  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

CASES = [  # name, config, batch, seed, random_pose, store_full
    ("tiny_randpose", "tiny", 2, 11, True, True),
    ("tiny_level", "tiny", 1, 12, False, True),
    ("plumbing", "plumbing", 1, 0, False, True),
    ("carla_res", "carla_res", 1, 3, True, False),
    ("lift_splat", "lift_splat", 1, 0, False, False),
    ("perceive", "perceive", 1, 0, False, False),
    # BASELINE configs[4]: 400x400 BEV, D=96, C=128, S=5 (4.8 M frustum points), non-level cameras
    ("stress", "stress", 1, 5, True, False),
]


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_reference(ref, cfg, inp):
    """get_geometry -> softmax (x) context -> projection_to_birds_eye_view, exactly as
    STP3.calculate_birds_eye_view_features does (stp3.py:303-318), entering after the Encoder."""
    B, S, N = inp["feat"].shape[:3]
    fake = make_fake_stp3(ref, cfg.x_bound, cfg.y_bound, cfg.z_bound, cfg.d_bound, cfg.final_dim,
                          cfg.downsample, cfg.discount)
    STP3 = ref.stp3.STP3
    pack = ref.network.pack_sequence_dim
    geom = STP3.get_geometry(fake, pack(inp["intrinsics"]), pack(inp["extrinsics"]))
    geom = ref.network.unpack_sequence_dim(geom, B, S)
    depth_prob = pack(pack(inp["depth_logits"])).softmax(dim=1)
    feat = pack(pack(inp["feat"]))
    x = depth_prob.unsqueeze(1) * feat.unsqueeze(2)                       # stp3.py:216
    x = x.view(B, S, N, *x.shape[1:]).permute(0, 1, 2, 4, 5, 6, 3)        # stp3.py:220-221
    bev = STP3.projection_to_birds_eye_view(fake, x, geom, inp["future_egomotion"])  # mutates geom
    # voxel index / mask / rank with the reference's own expressions (stp3.py:287-289, 239-255)
    idx = ((geom - (fake.bev_start_position - fake.bev_resolution / 2.0)) / fake.bev_resolution).long()
    dim = fake.bev_dimension
    keep = ((idx[..., 0] >= 0) & (idx[..., 0] < dim[0]) & (idx[..., 1] >= 0) & (idx[..., 1] < dim[1])
            & (idx[..., 2] >= 0) & (idx[..., 2] < dim[2]))
    rank = idx[..., 0] * (dim[1] * dim[2]) + idx[..., 1] * dim[2] + idx[..., 2]
    rank = torch.where(keep, rank, torch.full_like(rank, -1)).to(torch.int32)
    return fake, geom, rank, bev


def main():
    os.makedirs(OUT, exist_ok=True)
    ref = load_reference()
    only = set(sys.argv[1:])                      # optional: regenerate just the named cases
    for name, cfg_name, batch, seed, rp, full in CASES:
        if only and name not in only:
            continue
        cfg = syn.CONFIGS[cfg_name]
        inp = syn.lift_inputs(cfg, batch, seed=seed, random_pose=rp)
        fake, geom, rank, bev = run_reference(ref, cfg, inp)
        # host parameters as evaluated by the reference's calls in this container
        rot, trans = inp["extrinsics"][..., :3, :3], inp["extrinsics"][..., :3, 3]
        cam_M = rot.matmul(torch.inverse(inp["intrinsics"]))
        pose = ref.geometry.pose_vec2mat(inp["future_egomotion"])
        fr = fake.frustum
        rec = dict(
            config=cfg_name, batch=batch, seed=seed, random_pose=rp,
            intrinsics=inp["intrinsics"].numpy(), extrinsics=inp["extrinsics"].numpy(),
            future_egomotion=inp["future_egomotion"].numpy(),
            cam_M=cam_M.numpy(), cam_t=trans.contiguous().numpy(),
            ego_R=pose[..., :3, :3].contiguous().numpy(), ego_t=pose[..., :3, 3].contiguous().numpy(),
            xs=fr[0, 0, :, 0].contiguous().numpy(), ys=fr[0, :, 0, 1].contiguous().numpy(),
            ds=fr[:, 0, 0, 2].contiguous().numpy(),
            bev_resolution=fake.bev_resolution.numpy(), bev_start_position=fake.bev_start_position.numpy(),
            bev_dimension=fake.bev_dimension.numpy(),
            bev_offset=(fake.bev_start_position - fake.bev_resolution / 2.0).numpy(),
            feat_sha=sha(inp["feat"].numpy()), depth_sha=sha(inp["depth_logits"].numpy()),
            rank_sha=sha(rank.numpy()), geom_sha=sha(geom.numpy()),
            n_kept=int((rank >= 0).sum()),
            bev_tc_sum=bev.double().sum(dim=(-1, -2)).numpy(),
        )
        if full:
            rec.update(feat=inp["feat"].numpy(), depth_logits=inp["depth_logits"].numpy(),
                       rank=rank.numpy(), bev=bev.numpy())
            if geom.numel() < 200_000:
                rec["geom"] = geom.numpy()
        else:
            g = torch.Generator().manual_seed(1234)
            flat = bev.reshape(-1)
            nz = torch.nonzero(flat).squeeze(1)
            pick_nz = nz[torch.randint(0, nz.numel(), (30_000,), generator=g)]
            pick_any = torch.randint(0, flat.numel(), (10_000,), generator=g)
            pick = torch.cat([pick_nz, pick_any])
            rec.update(bev_sample_index=pick.numpy(), bev_sample_value=flat[pick].numpy())
        path = os.path.join(OUT, f"lift_splat_{name}.npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: kept {rec['n_kept']} / {rank.numel()} points  -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
