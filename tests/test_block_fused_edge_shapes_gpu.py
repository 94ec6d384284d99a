"""The back-to-back TemporalBlock tail (stp3_block_fused_fwd) at the edges of its tile schedule, for both chain layouts
(block 1: three 35-channel paths + projection + ego-motion biases; block 2: block-diagonal chain + identity residual):
a map of one 8x16 tile, a map with fewer tiles than SMs, a narrow 200x24 map, and a map whose last tile row and column
are ragged.  Against the fp64 oracle and the unfused launch sequence; plus bitwise repeatability of both launches."""
import copy

import pytest
import torch

from oracle import torch_dense as TD
from oracle.make_golden_dense import dense_input
from stp3_b200 import dense
from stp3_b200.models.temporal_model import TemporalModel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(x, B, H, W, fused, monkeypatch):
    monkeypatch.setenv("STP3_BLOCK_FUSED", fused)
    tm = TD.init_exact(TemporalModel(70, 3, (H, W), start_out_channels=64), seed=42).eval()
    ref = copy.deepcopy(tm).double()
    tm = tm.to(DEV)
    tm.model[0].n_const = 6
    const = x[:, :, 64:, 0, 0].reshape(B * 3, 6).contiguous().to(DEV)
    y = dense.to_f32(tm.forward_hl(dense.from_f32(x[:, :, :64].contiguous().to(DEV)), const=const), 0, 64)
    assert ("tail" in tm.model[0].packed()) == (fused == "1") and ("tail" in tm.model[1].packed()) == (fused == "1")
    return y, ref, tm, const


@pytest.mark.parametrize("B,H,W", [
    (1, 8, 16),       # one tile per image
    (1, 40, 48),      # 5 x 3 tiles per image: fewer tiles than SMs
    (2, 200, 24),     # narrow map, ragged last tile column
    (1, 37, 53),      # ragged last tile row and column
])
def test_block_fused_edge_shapes_vs_oracle(B, H, W, monkeypatch):
    x = dense_input((B, 3, 70, H, W), 41)
    x[:, :, 64:] = x[:, :, 64:, :1, :1]                        # the six ego-motion channels are spatially constant
    with torch.no_grad():
        y, ref_tm, _, _ = _run(x, B, H, W, "1", monkeypatch)
        ref = TD.temporal_model(x.double(), ref_tm)
        y0, _, _, _ = _run(x, B, H, W, "0", monkeypatch)
    scale = ref.abs().max().item()
    err = (y.double().cpu() - ref).abs().max().item()
    assert err <= 1e-3 * scale, (err, scale)
    assert (y - y0).abs().max() <= 5e-5 * y0.abs().max(), "fused and unfused block tails disagree"
    print(f"block fused {B}x{H}x{W}: {err / scale:.2e} of max vs fp64 oracle")


def test_block_fused_deterministic(monkeypatch):
    """Two launches of each block give bitwise-identical outputs and column sums at the perceive map size."""
    monkeypatch.setenv("STP3_BLOCK_FUSED", "1")
    B, H, W = 2, 200, 200
    x = dense_input((B, 3, 70, H, W), 5)
    x[:, :, 64:] = x[:, :, 64:, :1, :1]
    calls = []
    orig = dense.block_tail

    def rec(*a, **k):
        calls.append((a, k))
        return orig(*a, **k)
    monkeypatch.setattr(dense, "block_tail", rec)
    with torch.no_grad():
        _run(x, B, H, W, "1", monkeypatch)
        assert len(calls) == 2
        for a, k in calls:
            sums = [None, None]
            outs = []
            for i in range(2):
                kk = dict(k)
                if k.get("col_sums") is not None:
                    sums[i] = torch.empty_like(k["col_sums"])
                    kk["col_sums"] = sums[i]
                outs.append(orig(*a, **kk))
            assert torch.equal(outs[0].hi, outs[1].hi) and torch.equal(outs[0].lo, outs[1].lo)
            if sums[0] is not None:
                assert torch.equal(sums[0], sums[1])
