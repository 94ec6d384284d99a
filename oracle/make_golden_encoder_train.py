"""Generates tests/golden/encoder_heads_train.npz from the UNMODIFIED reference UpsamplingConcat and the two encoder
heads built from the reference's modules the way its Encoder builds them for efficientnet-b4 at downsample 8
(stp3/models/encoder.py: DeepLabHead(160, 160, hidden 64) -> UpsamplingConcat(160 + 56, C or D)), run in train mode, fp32
on the CPU of the build container, with seeded weights (init_exact), endpoints and upstream gradients.  Each DeepLab
head's Dropout is replaced by a fixed keep mask as in oracle/make_golden_head_train.py.  Test infrastructure; run by
hand:
    python -m oracle.make_golden_encoder_train

Records, each stored like deeplab_train_*.npz under a prefix: "uc." the UpsamplingConcat(216, 64) alone on seeded
x_to_upsample (4, 160, 14, 30) / x (4, 56, 28, 60); "feat." and "depth." the two heads (C = 64, D = 48) on the same seeded
r_lo (4, 56, 28, 60) / r_hi (4, 160, 14, 30).  BatchNorm momentum 0.05.
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
M, C_LO, C_HI, H, W = 4, 56, 160, 14, 30          # r_hi (M, C_HI, H, W), r_lo (M, C_LO, 2H, 2W)
HIDDEN, C_FEAT, D_DEPTH = 64, 64, 48
MOMENTUM = 0.05
SEEDS = {"uc": 3, "feat": 4, "depth": 6}           # init_exact seed of each record's modules
LO_SEED, HI_SEED, GRAD_SEED, MASK_SEED = 5, 7, 9, 11
N_OUT, N_GRAD = 4096, 512
RELU_NEAR = 1e-4


def endpoints():
    r_lo = TD.exact_gauss((M, C_LO, 2 * H, 2 * W), torch.Generator().manual_seed(LO_SEED))
    r_hi = TD.exact_gauss((M, C_HI, H, W), torch.Generator().manual_seed(HI_SEED))
    return r_lo, r_hi


def make_modules(conv_module, name):
    """(DeepLabHead or None, UpsamplingConcat) of record `name` from the module namespace conv_module (the reference's
    stp3.layers.convolutions, or this package's), seeded, train mode."""
    cout = D_DEPTH if name == "depth" else C_FEAT
    mods = torch.nn.ModuleList([conv_module.UpsamplingConcat(C_HI + C_LO, cout)])
    if name != "uc":
        mods.insert(0, conv_module.DeepLabHead(C_HI, C_HI, hidden_channel=HIDDEN))
    TD.init_exact(mods, seed=SEEDS[name])
    for m in mods.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = MOMENTUM
    mods.train()
    return (mods[0] if name != "uc" else None), mods[-1], mods


def main():
    ref = load_reference()
    rec = {"shape": np.array((M, C_LO, C_HI, H, W)), "momentum": MOMENTUM, "mask_seed": MASK_SEED}
    for name in SEEDS:
        head, up, mods = make_modules(ref.convolutions, name)
        r_lo, r_hi = endpoints()
        r_lo.requires_grad_(True), r_hi.requires_grad_(True)
        if head is not None:
            p = head[0].project[3].p
            head[0].project[3] = FixedDropout(TH.dropout_keep_mask((M, HIDDEN, H, W), MASK_SEED, p), p)
            rec["p"] = p
        near = []

        def record(_, inp):
            t = inp[0].detach().reshape(-1)
            idx = torch.nonzero(t.abs() < RELU_NEAR * t.abs().max()).squeeze(1)
            near.append((idx.to(torch.int32).numpy(), (t[idx] > 0).numpy()))
        hooks = [m.register_forward_pre_hook(record) for m in mods.modules() if isinstance(m, torch.nn.ReLU)]
        out = up(head(r_hi) if head is not None else r_hi, r_lo)
        for h in hooks:
            h.remove()
        G = TT.upstream_grads({"out": out}, seed=GRAD_SEED)["out"]
        (out * G).sum().backward()
        pre = name + "."
        rec[pre + "n_relu"] = len(near)
        for k, (idx, pos) in enumerate(near):
            rec[f"{pre}relu{k}_idx"], rec[f"{pre}relu{k}_pos"] = idx, pos
        flat = out.detach().reshape(-1)
        rec[pre + "out_s"] = flat[TT.sample_index(pre + "out", flat.numel(), N_OUT)].numpy()
        rec[pre + "out_amax"] = float(flat.abs().max())
        for k, b in mods.named_buffers():
            if not k.endswith("mask"):
                rec[pre + k] = b.numpy()
        for k, prm in list(mods.named_parameters()) + [("r_lo", r_lo), ("r_hi", r_hi)]:
            flat = prm.grad.reshape(-1)
            rec[f"{pre}grad_{k}_s"] = flat[TT.sample_index(f"{pre}grad.{k}", flat.numel(), N_GRAD)].numpy()
            rec[f"{pre}grad_{k}_amax"] = float(flat.abs().max())
        print(name, tuple(out.shape), f"{len(near)} ReLU calls")
    path = os.path.join(OUT, "encoder_heads_train.npz")
    np.savez_compressed(path, **rec)
    print(f"{os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
