"""GPU: the back-to-back kernels' outputs (stp3_block_fused_fwd: both TemporalBlock tail layouts, with the projection
and with the identity residual; stp3_aspp_fused_fwd: the ASPP instance and the 3x3 -> classifier tail) on one-tile
maps, maps whose last tile row and column are ragged, and maps with several tiles per CTA, written through the TMA
store path.

The kernels compute every value with the same instructions whichever way the tile leaves the SM, so the hi / lo planes
and column sums are held bitwise to digests recorded from the build that stored them with per-thread global stores
(tests/golden/fused_tma_store_digests.json).  Each output is also held to the fp64 composition of the same operation
(tests/fused_cases.py), and output channels outside the written window keep their sentinel.

    python tests/test_fused_tma_store_gpu.py --write    # record the digests of the current build (on an H100)
"""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from stp3_b200 import dense  # noqa: E402
from tests import fused_cases as FC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIGESTS = os.path.join(ROOT, "tests", "golden", "fused_tma_store_digests.json")
SENT_HI = 7.0                                  # bf16-exact sentinel of the output channels outside the window
RATES = (12, 24, 36)

# (tag, layout, projection, B, T, H, W, seed)
BLOCK_CASES = [
    ("L0 projection, one tile", 0, True, 1, 3, 8, 16, 1),
    ("L1 identity, one tile", 1, False, 1, 3, 8, 16, 2),
    ("L0 projection, ragged 13x37", 0, True, 1, 3, 13, 37, 3),
    ("L1 identity, ragged 13x37", 1, False, 1, 3, 13, 37, 4),
    ("L0 identity, ragged 21x35", 0, False, 2, 1, 21, 35, 5),
    ("L1 projection, ragged 17x33", 1, True, 1, 2, 17, 33, 6),
    ("L0 projection, several tiles per CTA 75x197", 0, True, 1, 3, 75, 197, 7),
    ("L1 identity, several tiles per CTA 75x197", 1, False, 1, 3, 75, 197, 8),
]
# (tag, rates, cin, n_out, n_store, relu, out_cs, out_coff, B, T, H, W, seed)
ASPP_CASES = [
    ("ASPP, one tile", [None] + [(r, r) for r in RATES], 64, 128, 128, True, 128, 0, 1, 3, 8, 16, 11),
    ("ASPP, ragged 13x37", [None] + [(r, r) for r in RATES], 64, 128, 128, True, 128, 0, 1, 3, 13, 37, 12),
    ("ASPP, several tiles per CTA 75x197", [None] + [(r, r) for r in RATES], 64, 128, 128, True, 128, 0, 1, 2, 75, 197,
     13),
    ("ASPP, out_coff 16 of 160 channels, ragged", [None, (2, 2)], 64, 128, 128, True, 160, 16, 2, 1, 19, 35, 14),
    ("tail, n_store 64, no ReLU, one tile", [(1, 1)], 128, 40, 64, False, 64, 0, 1, 3, 8, 16, 15),
    ("tail, n_store 64, no ReLU, ragged 13x37", [(1, 1)], 128, 40, 64, False, 64, 0, 1, 3, 13, 37, 16),
    ("n_store 64 with ReLU, out_coff 16, several tiles per CTA", [None, (3, 3)], 64, 128, 64, True, 96, 16, 1, 3, 75,
     197, 17),
]


def _f64(h: dense.HL, c: int) -> torch.Tensor:
    return h.hi[..., :c].double() + h.lo[..., :c].double()


def _digest(t: torch.Tensor) -> str:
    t = t.contiguous().cpu()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def run_block(case):
    tag, layout, proj, B, T, H, W, seed = case
    bc = FC.block_case(layout, proj, seed=seed, dev=DEV)
    mid = FC.planes(B, T, H, W, 128, 128, seed=seed + 50, dev=DEV)
    x = FC.planes(B, T, H, W, 64, 64, seed=seed + 51, dev=DEV)
    n = B * T
    hid, ib = FC.rnd(n, 128, seed=seed + 52, scale=0.5, dev=DEV), FC.rnd(n, 64, seed=seed + 53, scale=0.5, dev=DEV)
    rb = FC.rnd(n, 64, seed=seed + 54, scale=0.5, dev=DEV) if proj else None
    sums = torch.full((n, 64), float("nan"), device=DEV)
    with torch.no_grad():
        y = dense.block_tail(mid, x, bc.pb, hid, ib, rb, col_sums=sums)
        torch.cuda.synchronize()
        ref = FC.block_direct(bc, _f64(mid, 128).permute(0, 4, 1, 2, 3), _f64(x, 64).permute(0, 4, 1, 2, 3), hid, ib,
                              rb).cpu()
    got = _f64(y, 64).reshape(n, H, W, 64).cpu()
    return {"hi": y.hi, "lo": y.lo, "col_sums": sums}, got, ref, ref.sum(dim=(1, 2))


def run_aspp(case):
    tag, rates, cin, n_out, n_store, relu, out_cs, out_coff, B, T, H, W, seed = case
    ac = FC.aspp_case(cin, rates, n_out=n_out, seed=seed, dev=DEV)
    x = FC.planes(B, T, H, W, cin, cin, seed=seed + 50, dev=DEV)
    n = B * T
    ib = FC.rnd(n, 128, seed=seed + 51, scale=0.5, dev=DEV)
    ib[:, n_out:] = 0
    out = dense.HL(torch.full((B, T, H, W, out_cs), SENT_HI, dtype=torch.bfloat16, device=DEV),
                   torch.zeros((B, T, H, W, out_cs), dtype=torch.bfloat16, device=DEV), out_cs)
    with torch.no_grad():
        dense.aspp_fused(x, ac.pa, ib, out=out, out_coff=out_coff, relu=relu, n_store=n_store)
        torch.cuda.synchronize()
        ref = FC.aspp_direct(ac, _f64(x, cin).reshape(n, H, W, cin).permute(0, 3, 1, 2), ib, relu)[..., :n_store].cpu()
    w = slice(out_coff, out_coff + n_store)
    outside = torch.ones(out_cs, dtype=torch.bool)
    outside[w] = False
    hi_out, lo_out = out.hi[..., outside], out.lo[..., outside]
    assert bool((hi_out == SENT_HI).all()) and bool((lo_out == 0).all()), "a channel outside the output window was written"
    got = (out.hi[..., w].double() + out.lo[..., w].double()).reshape(n, H, W, n_store).cpu()
    return {"hi": out.hi[..., w], "lo": out.lo[..., w]}, got, ref, None


def outputs():
    """{tag: {plane: digest}} of every case, after checking each against the fp64 composition"""
    res = {}
    for case, run in [(c, run_block) for c in BLOCK_CASES] + [(c, run_aspp) for c in ASPP_CASES]:
        planes, got, ref, ref_sums = run(case)
        scale = ref.abs().max().item()
        err = (got - ref).abs().max().item()
        assert err <= 1e-4 * scale, (case[0], err, scale)
        if ref_sums is not None:
            s = planes["col_sums"].double().cpu()
            assert (s - ref_sums).abs().max().item() <= 1e-4 * ref.abs().sum(dim=(1, 2)).max().item(), case[0]
        res[case[0]] = {k: _digest(v) for k, v in planes.items()}
    return res


def test_fused_outputs_bitwise_equal_to_recorded():
    with open(DIGESTS) as f:
        want = json.load(f)["digests"]
    got = outputs()
    assert set(got) == set(want), "the case list and the recorded digests differ"
    bad = [(tag, k) for tag in got for k in got[tag] if got[tag][k] != want[tag][k]]
    assert not bad, f"outputs differ bitwise from the recorded ones: {bad}"


if __name__ == "__main__":
    if sys.argv[1:] == ["--write"]:
        with open(DIGESTS, "w") as f:
            json.dump({"device": torch.cuda.get_device_name(0), "digests": outputs()}, f, indent=1)
            f.write("\n")
    else:
        sys.exit(pytest.main([__file__, "-q"]))
