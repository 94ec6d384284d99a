"""The back-to-back DeepLab head kernel (stp3_aspp_fused_fwd) at the edges of its tile schedule: a map of one 8x16
tile, a map with fewer tiles than SMs, a narrow map with an odd number of tile rows whose neighbouring tiles skip
different dilation-24 / 36 padding taps, and a map whose ragged last tile row repeats in every image.  Against the fp64
oracle and the unfused launch sequence; plus bitwise repeatability (the kernel has no atomics)."""
import copy

import pytest
import torch

from oracle import torch_dense as TD
from oracle.make_golden_dense import dense_input
from stp3_b200.layers.convolutions import DeepLabHead

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _head():
    return TD.init_exact(DeepLabHead(64, 64, hidden_channel=128), seed=17).eval()


@pytest.mark.parametrize("B,H,W", [
    (1, 8, 16),       # one tile
    (1, 24, 32),      # 3 x 2 tiles
    (5, 200, 24),     # narrow map, 25 tile rows: tile rows 2 / 3 and 20 / 21 differ on the dilation-24 / 36 skips
    (2, 72, 200),     # 9 tile rows per image, ragged last tile column
])
def test_aspp_fused_edge_shapes_vs_oracle(B, H, W, monkeypatch):
    monkeypatch.setenv("STP3_ASPP_FUSED", "1")
    with torch.no_grad():
        x = dense_input((B, 64, H, W), 18)
        head = _head()
        ref = TD.deeplab_head(x.double(), copy.deepcopy(head).double())
        head = head.to(DEV)
        y = head(x.to(DEV))
        assert "fused" in head.packed() and "tail" in head.packed()
        scale = ref.abs().max().item()
        err = (y.double().cpu() - ref).abs().max().item()
        assert err <= 1e-3 * scale, (err, scale)
        monkeypatch.setenv("STP3_ASPP_FUSED", "0")
        head2 = _head().to(DEV)
        y2 = head2(x.to(DEV))
        assert "fused" not in head2.packed()
        assert (y - y2).abs().max() <= 2e-5 * y2.abs().max(), "fused and unfused ASPP disagree"
    print(f"aspp fused {B}x{H}x{W}: {err / scale:.2e} of max vs fp64 oracle")


def test_aspp_fused_deterministic(monkeypatch):
    """Two launches give bitwise-identical outputs at the perceive map size."""
    monkeypatch.setenv("STP3_ASPP_FUSED", "1")
    with torch.no_grad():
        x = dense_input((3, 64, 200, 200), 5).to(DEV)
        head = TD.init_exact(DeepLabHead(64, 64, hidden_channel=128), seed=3).eval().to(DEV)
        a = head(x)
        b = head(x)
    assert torch.equal(a, b)
