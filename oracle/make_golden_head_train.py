"""Generates tests/golden/deeplab_train_*.npz from the UNMODIFIED reference DeepLabHead (stp3/layers/convolutions.py)
run in train mode, fp32 on the CPU of the build container, with seeded weights (init_exact), inputs and upstream
gradients.  The instance's ASPP.project[3] Dropout is replaced by a fixed keep mask, regenerated from MASK_SEED by
oracle.torch_deeplab_train.dropout_keep_mask rather than stored.  Test infrastructure; run by hand:
    python -m oracle.make_golden_head_train

Configurations: "temporal" = TemporalModel.final_conv, DeepLabHead(64, 64, hidden 128) on N = 6 BEV frames of 48x64;
"encoder" = the encoder's feature_layer_1, DeepLabHead(160, 160, hidden 64) on N = 4 maps of 14x30 (every dilated tap
but the centre reads only padding there).  BatchNorm momentum 0.05.  Stored like decoder_train_*.npz
(oracle/make_golden_train.py): out_s / out_amax, every buffer, grad_<param>_s / _amax, grad_x_s, relu<k>_idx / _pos.
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

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
# name -> (in_channels, num_classes, hidden, N, H, W)
CONFIGS = {"temporal": (64, 64, 128, 6, 48, 64), "encoder": (160, 160, 64, 4, 14, 30)}
MOMENTUM = 0.05
WEIGHT_SEED, INPUT_SEED, GRAD_SEED, MASK_SEED = 3, 5, 9, 11
N_OUT, N_GRAD = 4096, 512
RELU_NEAR = 1e-4


def make_head(DeepLabHead, cin, ncls, hidden):
    head = TD.init_exact(DeepLabHead(cin, ncls, hidden_channel=hidden), seed=WEIGHT_SEED)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = MOMENTUM
    return head.train()


class FixedDropout(torch.nn.Module):
    """Dropout with a given keep mask (scaled by 1 / (1 - p) like nn.Dropout in train mode)."""

    def __init__(self, mask, p):
        super().__init__()
        self.mask, self.p = mask, p

    def forward(self, x):
        return x * self.mask.to(x.dtype) * (1.0 / (1.0 - self.p))


def main():
    ref = load_reference()
    for name, (cin, ncls, hidden, N, H, W) in CONFIGS.items():
        head = make_head(ref.convolutions.DeepLabHead, cin, ncls, hidden)
        p = head[0].project[3].p
        head[0].project[3] = FixedDropout(TH.dropout_keep_mask((N, hidden, H, W), MASK_SEED, p), p)
        x = TD.exact_gauss((N, cin, H, W), torch.Generator().manual_seed(INPUT_SEED)).requires_grad_(True)
        near = []

        def record(_, inp):
            t = inp[0].detach().reshape(-1)
            idx = torch.nonzero(t.abs() < RELU_NEAR * t.abs().max()).squeeze(1)
            near.append((idx.to(torch.int32).numpy(), (t[idx] > 0).numpy()))
        hooks = [m.register_forward_pre_hook(record) for m in head.modules() if isinstance(m, torch.nn.ReLU)]
        out = head(x)
        for h in hooks:
            h.remove()
        G = TT.upstream_grads({"out": out}, seed=GRAD_SEED)["out"]
        (out * G).sum().backward()
        rec = {"shape": np.array((N, cin, H, W)), "cfg": np.array((cin, ncls, hidden)), "momentum": MOMENTUM,
               "p": p, "mask_seed": MASK_SEED, "n_relu": len(near)}
        for k, (idx, pos) in enumerate(near):
            rec[f"relu{k}_idx"], rec[f"relu{k}_pos"] = idx, pos
        flat = out.detach().reshape(-1)
        rec["out_s"] = flat[TT.sample_index("out", flat.numel(), N_OUT)].numpy()
        rec["out_amax"] = float(flat.abs().max())
        for k, b in head.named_buffers():
            if not k.endswith("mask"):
                rec[k] = b.numpy()
        for k, prm in list(head.named_parameters()) + [("x", x)]:
            flat = prm.grad.reshape(-1)
            rec[f"grad_{k}_s"] = flat[TT.sample_index(f"grad.{k}", flat.numel(), N_GRAD)].numpy()
            rec[f"grad_{k}_amax"] = float(flat.abs().max())
        path = os.path.join(OUT, f"deeplab_train_{name}.npz")
        np.savez_compressed(path, **rec)
        print(name, f"{os.path.getsize(path) / 1e3:.0f} kB", tuple(out.shape), f"{len(near)} ReLU calls")


if __name__ == "__main__":
    main()
