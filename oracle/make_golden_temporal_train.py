"""Generates tests/golden/temporal_train_*.npz from the UNMODIFIED reference TemporalModel (stp3/models/temporal_model.py)
run in train mode, fp32 on the CPU of the build container, with seeded weights (init_exact on this package's
TemporalModel, loaded into the reference's with strict=True), inputs and upstream gradients.  The head's
ASPP.project[3] Dropout is replaced by a fixed keep mask, regenerated from MASK_SEED by
oracle.torch_deeplab_train.dropout_keep_mask rather than stored (as oracle/make_golden_head_train.py does).  Test
infrastructure; run by hand:
    python -m oracle.make_golden_temporal_train

Configurations: "perceive" = TemporalModel(70, receptive field 3, (48, 64)) on B = 2 (64 BEV channels + the 6 ego-motion
channels, which the reference sees broadcast); "stress" = TemporalModel(134, receptive field 5, (16, 24)) on B = 1.
BatchNorm momentum 0.05.  Stored like deeplab_train_*.npz: out_s / out_amax, every buffer, grad_<param>_s / _amax,
grad_x_s / _amax, relu<k>_idx / _pos (the ReLU inputs within round-off of zero and their sign in the reference).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle import torch_dense as TD  # noqa: E402
from oracle import torch_dense_train as TT  # noqa: E402
from oracle import torch_deeplab_train as TH  # noqa: E402
from oracle.make_golden_head_train import FixedDropout  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
# name -> (in_channels, receptive field S, B, H, W)
CONFIGS = {"perceive": (70, 3, 2, 48, 64), "stress": (134, 5, 1, 16, 24)}
MOMENTUM = 0.05
WEIGHT_SEED, INPUT_SEED, GRAD_SEED, MASK_SEED = 3, 5, 9, 11
N_OUT, N_GRAD = 4096, 512
RELU_NEAR = 1e-4


def make_models(TemporalModelRef, cin, S, H, W):
    """(this package's TemporalModel, the reference's) with the same seeded weights, momentum MOMENTUM, in train()."""
    from stp3_b200.models.temporal_model import TemporalModel
    ours = TD.init_exact(TemporalModel(cin, S, (H, W), start_out_channels=64), seed=WEIGHT_SEED)
    ref = TemporalModelRef(cin, S, (H, W), start_out_channels=64)
    ref.load_state_dict(ours.state_dict(), strict=True)
    for m in list(ours.modules()) + list(ref.modules()):
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = MOMENTUM
    return ours.train(), ref.train()


def main():
    ref_pkg = load_reference()
    for name, (cin, S, B, H, W) in CONFIGS.items():
        _, tm = make_models(ref_pkg.temporal_model.TemporalModel, cin, S, H, W)
        head = tm.final_conv
        hidden = head[0].project[0].out_channels
        p = head[0].project[3].p
        head[0].project[3] = FixedDropout(TH.dropout_keep_mask((B * S, hidden, H, W), MASK_SEED, p), p)
        x = TD.exact_gauss((B, S, cin, H, W), torch.Generator().manual_seed(INPUT_SEED)).requires_grad_(True)
        near = []

        def record(_, inp):
            t = inp[0].detach().reshape(-1)
            idx = torch.nonzero(t.abs() < RELU_NEAR * t.abs().max()).squeeze(1)
            near.append((idx.to(torch.int32).numpy(), (t[idx] > 0).numpy()))
        hooks = [m.register_forward_pre_hook(record) for m in tm.modules() if isinstance(m, torch.nn.ReLU)]
        out = tm(x)
        for h in hooks:
            h.remove()
        G = TT.upstream_grads({"out": out}, seed=GRAD_SEED)["out"]
        (out * G).sum().backward()
        rec = {"shape": np.array((B, S, cin, H, W)), "momentum": MOMENTUM, "p": p, "mask_seed": MASK_SEED,
               "hidden": hidden, "n_relu": len(near)}
        for k, (idx, pos) in enumerate(near):
            rec[f"relu{k}_idx"], rec[f"relu{k}_pos"] = idx, pos
        flat = out.detach().reshape(-1)
        rec["out_s"] = flat[TT.sample_index("out", flat.numel(), N_OUT)].numpy()
        rec["out_amax"] = float(flat.abs().max())
        for k, b in tm.named_buffers():
            if not k.endswith("mask"):
                rec[k] = b.numpy()
        for k, prm in list(tm.named_parameters()) + [("x", x)]:
            flat = prm.grad.reshape(-1)
            rec[f"grad_{k}_s"] = flat[TT.sample_index(f"grad.{k}", flat.numel(), N_GRAD)].numpy()
            rec[f"grad_{k}_amax"] = float(flat.abs().max())
        path = os.path.join(OUT, f"temporal_train_{name}.npz")
        np.savez_compressed(path, **rec)
        print(name, f"{os.path.getsize(path) / 1e3:.0f} kB", tuple(out.shape), f"{len(near)} ReLU calls")


if __name__ == "__main__":
    main()
