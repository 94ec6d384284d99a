"""GPU: the convolutions of one TemporalModel train step under the stp3_conv_fwd contract of tests/test_conv_contract_gpu.py.

Every dense.conv call of a forward and backward of TemporalModel(70 -> 64, S = 3, 6 ego-motion channels) with its
blocks and head in train mode is recorded: the 1x1x1 entry / projection / aggregation convolutions with per-image
biases, the causal (2,3,3) / (1,3,3) raw convolutions, their input gradients with anti-causal time taps (time offset
+1, frames at or past T read as zero), the transposed 1x1x1 of the input gradient and the head's.  Each call is
replayed with tune = (0, 0) and with every candidate dense.tune_candidates offers, into sentinel-filled outputs, and
checked with that file's bars: against the exact fp64 convolution of the stored planes (3e-5 of max) and against the
fp64 three-product model per element (2^-17 split allowance + model_bar(K)); nothing outside the written window
changed; a second launch is bitwise identical."""
import torch

from oracle import torch_dense as TD
from stp3_b200 import dense
from stp3_b200.models.temporal_model import TemporalModel
from tests import test_conv_contract_gpu as CC

pytestmark = CC.pytestmark
DEV = CC.DEV


def record_train_step():
    tm = TD.init_exact(TemporalModel(70, 3, (16, 24), start_out_channels=64), seed=3)
    tm.model[0].n_const = 6
    tm = tm.train().to(DEV)
    x = TD.exact_gauss((2, 3, 64, 16, 24), torch.Generator().manual_seed(5)).to(DEV).requires_grad_(True)
    const = TD.exact_gauss((6, 6), torch.Generator().manual_seed(6)).to(DEV)
    torch.manual_seed(0)
    with CC.Recorder("temporal_train") as rec:
        tm(x, const=const).square().sum().backward()
    return rec.calls


def test_train_step_convolutions_under_every_tiling():
    calls = record_train_step()
    taps = [c.pc.taps for c in calls]
    assert any(any(dt > 0 for dt, _, _ in t) for t in taps), "no anti-causal input-gradient convolution recorded"
    assert any(any(dt < 0 for dt, _, _ in t) for t in taps), "no causal 3-D convolution recorded"
    bad, n = [], 0
    for i, call in enumerate(calls):
        exact, model, scale = CC.references(call)
        worst = [0.0, 0.0]
        for cfg in [(0, 0)] + dense.tune_candidates(call.pc):
            got, same, untouched = CC.replay(call, cfg)
            assert set(got) == set(exact), (set(got), set(exact))
            e_x = max(float((got[k] - exact[k].reshape(got[k].shape)).abs().max()) / scale[k] for k in got)
            e_m = max(CC._excess(got[k], model[k].reshape(got[k].shape), CC.SPLIT if k in ("y", "y2") else 0.0) /
                      scale[k] for k in got)
            bar = CC.model_bar(len(call.pc.taps) * call.pc.cin_p)
            worst = [max(worst[0], e_x), max(worst[1], e_m)]
            n += 1
            if not (e_x <= CC.EXACT_BAR and e_m <= bar and same and untouched):
                bad.append((i, cfg, e_x, e_m, bar, same, untouched))
        t = call.pc.taps
        print(f"  #{i:<3d} {len(t)}tap dt {sorted({d for d, _, _ in t})} cin{call.pc.cin_p} bn{call.pc.bn} "
              f"{call.kw['geom']}  exact {worst[0]:.2e}  model {worst[1]:.2e}")
        del exact, model
    print(f"temporal train step: {len(calls)} convolutions, {n} replays")
    assert not bad, bad
