"""GPU: the convolutions of the DeepLab head's and the encoder heads' train steps under the stp3_conv_fwd contract of
tests/test_conv_contract_gpu.py.

Every dense.conv call of a forward and backward is recorded: the ASPP branches (dilations 12 / 24 / 36, taps partly or
wholly in the padding), their input gradients with mirrored dilated taps, the pooling branch's per-image bias
(img_bias) added to the input gradient, the 3x3 / 1x1 tail and the UpsamplingConcat convolutions with their input
gradients.  Each call is replayed with tune = (0, 0) and with every candidate dense.tune_candidates offers, into
sentinel-filled outputs, and checked with that file's bars: against the exact fp64 convolution of the stored planes
(3e-5 of max) and against the fp64 three-product model per element (2^-17 split allowance + model_bar(K)); nothing
outside the written window changed; a second launch is bitwise identical."""
import pytest
import torch

from stp3_b200 import dense
from tests import test_conv_contract_gpu as CC
from tests import test_train_contract_gpu as TC

pytestmark = CC.pytestmark


def record(step):
    with CC.Recorder("head train") as rec:
        step()
    return rec.calls


def deeplab_step(cin, ncls, hidden, N, H, W):
    from oracle import torch_dense as TD
    from stp3_b200.layers.convolutions import DeepLabHead
    head = TD.init_exact(DeepLabHead(cin, ncls, hidden_channel=hidden), seed=3).train().to(CC.DEV)
    x = TC.gauss((N, cin, H, W), 4).to(CC.DEV).requires_grad_(True)
    torch.manual_seed(5)
    return lambda: TC._step(lambda: head(x), 6)


def encoder_heads_step(name):
    from oracle import make_golden_encoder_train as MG
    from stp3_b200.layers import convolutions as CV
    head, up, mods = MG.make_modules(CV, name)
    mods.to(CC.DEV)
    r_lo, r_hi = (t.to(CC.DEV).requires_grad_(True) for t in MG.endpoints())
    torch.manual_seed(17)
    return lambda: TC._step(lambda: up(head(r_hi) if head is not None else r_hi, r_lo), 18)


STEPS = {
    "deeplab_temporal_48x64": lambda: deeplab_step(64, 64, 128, 6, 48, 64),
    "deeplab_encoder_14x30": lambda: deeplab_step(160, 160, 64, 18, 14, 30),
    "encoder_heads_feat": lambda: encoder_heads_step("feat"),
    "encoder_heads_depth": lambda: encoder_heads_step("depth"),
}


@pytest.mark.parametrize("name", list(STEPS))
def test_train_step_convolutions_under_every_tiling(name):
    calls = record(STEPS[name]())
    bad, n, feats = [], 0, set()
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
            feats |= CC.features(call, cfg)
            n += 1
            if not (e_x <= CC.EXACT_BAR and e_m <= bar and same and untouched):
                bad.append((i, cfg, e_x, e_m, bar, same, untouched))
        print(f"  #{i:<3d} {len(call.pc.taps)}tap cin{call.pc.cin_p} bn{call.pc.bn} {call.kw['geom']}  "
              f"exact {worst[0]:.2e}  model {worst[1]:.2e}")
        del exact, model
    print(f"{name}: {len(calls)} convolutions, {n} replays")
    if name.startswith("deeplab"):
        assert "img_bias" in feats and any(len(c.pc.taps) == 9 and max(abs(t[1]) for t in c.pc.taps) >= 12
                                           for c in calls), feats
    assert not bad, bad
