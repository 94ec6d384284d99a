"""Shared helpers for the parity tests (test infrastructure)."""
import hashlib
import os

import numpy as np

from stp3_b200.utils import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LIFT_CASES = ["tiny_randpose", "tiny_level", "plumbing", "carla_res", "lift_splat", "perceive", "stress"]


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load_lift_case(name):
    """Fixture + regenerated (machine-independent) inputs; asserts the inputs hash to the recorded value."""
    g = dict(np.load(os.path.join(GOLDEN, f"lift_splat_{name}.npz"), allow_pickle=False))
    cfg = syn.CONFIGS[str(g["config"])]
    inp = syn.lift_inputs(cfg, int(g["batch"]), seed=int(g["seed"]), random_pose=bool(g["random_pose"]))
    assert sha(inp["feat"].numpy()) == str(g["feat_sha"]), "synthetic generator is not reproducing the fixture inputs"
    assert sha(inp["depth_logits"].numpy()) == str(g["depth_sha"])
    return cfg, inp, g


E2E_CASES = ["level", "tilted"]
E2E_KEYS = ("segmentation", "pedestrian", "hdmap")


def load_e2e_case(name):
    """tests/golden/e2e_perceive_<name>.npz (oracle/make_golden_e2e.py: the reference end to end at the headline size)
    + the regenerated single-sample inputs it was recorded on."""
    g = dict(np.load(os.path.join(GOLDEN, f"e2e_perceive_{name}.npz"), allow_pickle=False))
    cfg = syn.CONFIGS[str(g["config"])]
    inp = syn.lift_inputs(cfg, 1, seed=int(g["seed"]), tilt_deg=float(g["tilt_deg"]))
    assert sha(inp["feat"].numpy()) == str(g["feat_sha"]), "synthetic generator is not reproducing the fixture inputs"
    assert sha(inp["depth_logits"].numpy()) == str(g["depth_sha"])
    return cfg, inp, g


def e2e_errors(g, key, tensor):
    """(error vs the fp64 oracle, error vs the reference's fp32 output), both as a fraction of max |value|, on the
    fixture's 12k-entry sample of output `key`; tensor = this implementation's full output for ONE sample."""
    flat = np.asarray(tensor, dtype=np.float64).reshape(-1)
    got = flat[g[f"{key}_index"]]
    m = float(g[f"{key}_max"])
    return (float(np.abs(got - g[f"{key}_oracle"]).max()) / m,
            float(np.abs(got - g[f"{key}_ref"].astype(np.float64)).max()) / m)
