"""Generates tests/golden/trunk_*.npz from the UNMODIFIED reference Encoder (oracle/ref_loader.py), CPU, fp32:

  Encoder.__init__ (with the fp32 restated trunk of oracle/efficientnet_oracle.py returned where it calls
  EfficientNet.from_pretrained; seeded synthetic weights), delete_unused_layers, then get_features_depth -- the
  reference's own endpoint bookkeeping (encoder.py:57-86) and both heads.  The endpoints are the inputs its heads
  receive (forward pre-hooks on feature_layer_1 / feature_layer_2).

  trunk_b4_224x480.npz   one 224x480 image
  trunk_b4_batch.npz     three 64x128 images

This pins the endpoint choice and the heads on this trunk to the reference code; the trunk's own arithmetic is pinned
only to the restatement (efficientnet-pytorch itself is not available).
Test infrastructure; run by hand:  python -m oracle.make_golden_trunk"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import efficientnet_oracle as EO  # noqa: E402
from oracle import torch_dense as TD  # noqa: E402
from oracle.make_golden_dense import dense_input  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
TRUNK_SEED, HEAD_SEED = 41, 42
CASES = {"trunk_b4_224x480": ((1, 3, 224, 480), 43), "trunk_b4_batch": ((3, 3, 64, 128), 44)}
HEADS = ("feature_layer_1", "feature_layer_2", "depth_layer_1", "depth_layer_2")


def make_trunk():
    """The full fp32 b4 restatement with the seeded weights the fixtures use (as EfficientNet.from_pretrained returns
    it: the reference's delete_unused_layers truncates it)."""
    return EO.init_random(EO.EfficientNetOracle('b4'), seed=TRUNK_SEED).eval()


def init_heads(enc):
    """Machine-independent head weights, keyed by module name (the reference's and the drop-in's names agree)."""
    for i, name in enumerate(HEADS):
        TD.init_exact(getattr(enc, name), seed=HEAD_SEED + i)
    return enc


def reference_encoder(ref):
    """The reference Encoder, built by its own unmodified __init__ around the restated trunk."""
    trunk = make_trunk()
    ref.encoder.EfficientNet = SimpleNamespace(from_pretrained=lambda name: trunk)
    cfg = SimpleNamespace(OUT_CHANNELS=64, USE_DEPTH_DISTRIBUTION=True, DOWNSAMPLE=8, NAME='efficientnet-b4')
    return init_heads(ref.encoder.Encoder(cfg, D=48)).eval()


def run(enc, img):
    """(reduction_3, reduction_4, feature, depth) of the reference's get_features_depth."""
    seen = {}

    def keep(key, i):
        def hook(module, args):
            seen.setdefault(key, args[i])          # returns None: the call's arguments are unchanged
        return hook
    hooks = [enc.feature_layer_1.register_forward_pre_hook(keep("r4", 0)),
             enc.feature_layer_2.register_forward_pre_hook(keep("r3", 1))]
    feat, depth = enc.get_features_depth(img)
    for h in hooks:
        h.remove()
    return seen["r3"], seen["r4"], feat, depth


def main():
    ref = load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    with torch.no_grad():
        enc = reference_encoder(ref)
        assert len(enc.backbone._blocks) == 22
        for name, (shape, seed) in CASES.items():
            r3, r4, feat, depth = run(enc, dense_input(shape, seed))
            np.savez_compressed(os.path.join(OUT, name + ".npz"), reduction_3=r3.numpy(), reduction_4=r4.numpy(),
                                feature=feat.numpy(), depth=depth.numpy(), in_seed=seed, shape=np.array(shape))
            print(name, tuple(r3.shape), tuple(r4.shape), tuple(feat.shape), tuple(depth.shape),
                  float(r4.abs().max()), float(feat.abs().max()))


if __name__ == "__main__":
    main()
