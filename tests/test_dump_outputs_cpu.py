"""CPU: bench.py --dump-outputs writes float32 .npy files of the timed step's outputs, skips heads that are None, keeps
a fixed seeded sample under the size limit, and writes the same files from run to run."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def outputs():
    return {"seg": torch.arange(1000, dtype=torch.float32).reshape(10, 100), "depth": torch.linspace(0, 1, 500, dtype=torch.float64),
            "instance": None}


def test_full_outputs_when_under_the_limit(tmp_path):
    bench.dump_outputs(outputs(), str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == ["depth.npy", "seg.npy"]
    seg, depth = np.load(tmp_path / "seg.npy"), np.load(tmp_path / "depth.npy")
    assert seg.dtype == np.float32 and depth.dtype == np.float32
    assert np.array_equal(seg, outputs()["seg"].numpy()) and np.allclose(depth, outputs()["depth"].numpy())


def test_seeded_sample_fits_the_limit_and_repeats(tmp_path):
    limit = 2000                                             # 1500 entries = 6000 bytes in all: sampled
    bench.dump_outputs(outputs(), str(tmp_path / "a"), limit=limit)
    bench.dump_outputs(outputs(), str(tmp_path / "b"), limit=limit)
    arrays = {}
    for name in ("seg", "depth"):
        a, b = np.load(tmp_path / "a" / f"{name}.npy"), np.load(tmp_path / "b" / f"{name}.npy")
        assert a.dtype == np.float32 and np.array_equal(a, b)
        arrays[name] = a
    assert sum(a.nbytes for a in arrays.values()) <= limit
    seg = arrays["seg"]                                      # entries of arange: the sampled indices, sorted and distinct
    assert len(seg) > 0 and np.all(np.diff(seg) > 0) and set(seg) <= set(range(1000))
    assert not os.path.exists(tmp_path / "a" / "instance.npy")
