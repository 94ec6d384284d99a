"""GPU: the EfficientNet trunk's convolutions under the stp3_conv_fwd contract of tests/test_conv_contract_gpu.py.

The expand (swish epilogue) and gated projection (per-image weights, w_img_stride; res_mode 1 for the identity skip)
calls of one b4 forward are recorded from the model and replayed with tune = (0, 0) and with every candidate
dense.tune_candidates offers for them (per_image for the projections: only streamed tilings, the stacked hi/lo operand
included), into sentinel-filled outputs.  Checked per replay, with that file's bars: every written value against the
exact fp64 convolution of the stored planes (3e-5 of max) and against the fp64 three-product model per element
(2^-17 split allowance + model_bar(K)); nothing outside the written channel windows changed; a second launch is
bitwise identical.  The fp64 reference evaluates image i with its own weights and applies swish after the epilogue."""
import dataclasses

import pytest
import torch

from oracle import efficientnet_oracle as EO
from stp3_b200 import dense
from stp3_b200.models import efficientnet as EN
from tests import conv_reference as R
from tests import test_conv_contract_gpu as CC

pytestmark = CC.pytestmark
DEV = CC.DEV


def record_trunk():
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=7), 'b4')
    nat = EN.EfficientNetTrunk('b4')
    nat.load_state_dict(ora.state_dict(), strict=True)
    nat = nat.to(DEV)
    torch.manual_seed(0)
    x = torch.randn(3, 3, 64, 128, device=DEV)
    with torch.no_grad(), CC.Recorder("trunk") as rec:
        nat.forward_hl(x)
    return rec.calls


def references(call: CC.Call):
    pc, kw = call.pc, call.kw
    stride = kw.get("w_img_stride", 0)
    args = dict(cin_off=kw.get("cin_off", 0), frames=kw.get("frames"), out_hw=kw.get("out_hw"))
    acc = {}
    for m in (False, True):
        if stride:
            nt, kbs = len(pc.taps), pc.cin_p // dense.KB
            n = nt * kbs * 2 * pc.bn * dense.KB
            parts = []
            for i in range(call.x.hi.shape[0]):
                wi = torch.as_strided(pc.w, (n,), (1,), pc.w.storage_offset() + i * stride)
                pci = dataclasses.replace(pc, w=wi.view(nt, kbs, 2, pc.bn, dense.KB))
                parts.append(R.tap_sum(call.x.hi[i:i + 1], call.x.lo[i:i + 1], pci, model=m, **args))
            acc[m] = torch.cat(parts)
        else:
            acc[m] = R.tap_sum(call.x.hi, call.x.lo, pc, model=m, **args)
    exact, model = R.epilogue(acc[False], pc, kw), R.epilogue(acc[True], pc, kw)
    if kw.get("swish"):
        for d in (exact, model):
            d["y"] = d["y"] * torch.sigmoid(d["y"])
    return exact, model, {k: max(float(v.abs().max()), 1e-20) for k, v in exact.items()}


def test_trunk_convolutions_under_every_tiling():
    calls = record_trunk()
    kinds = {"swish": 0, "per-image": 0, "per-image + res_mode 1": 0}
    cfgs_seen = {"swish": set(), "per-image": set()}
    bad, worst = [], {}
    for i, call in enumerate(calls):
        per_image = call.kw.get("w_img_stride", 0) > 0
        kind = "per-image" if per_image else "swish" if call.kw.get("swish") else None
        assert kind is not None, "the trunk launches only swish expand and per-image projection convolutions"
        kinds[kind] += 1
        kinds["per-image + res_mode 1"] += per_image and call.kw["residual"] is not None
        exact, model, scale = references(call)
        for cfg in [(0, 0)] + dense.tune_candidates(call.pc, per_image=per_image):
            cfgs_seen[kind].add((call.pc.bn, cfg))
            got, same, untouched = CC.replay(call, cfg)
            assert set(got) == set(exact), (set(got), set(exact))
            e_x = max(float((got[k] - exact[k].reshape(got[k].shape)).abs().max()) / scale[k] for k in got)
            e_m = max(CC._excess(got[k], model[k].reshape(got[k].shape), CC.SPLIT) / scale[k] for k in got)
            bar = CC.model_bar(len(call.pc.taps) * call.pc.cin_p)
            w = worst.setdefault(kind, [0.0, 0.0])
            w[0], w[1] = max(w[0], e_x), max(w[1], e_m)
            if not (e_x <= CC.EXACT_BAR and e_m <= bar and same and untouched):
                bad.append((i, kind, call.pc.bn, call.pc.cin_p, cfg, e_x, e_m, same, untouched))
        del exact, model
    print(f"\ntrunk: {len(calls)} convolutions {kinds}; worst (exact, beyond model): {worst}")
    assert not bad, bad
    assert all(kinds.values()), kinds
    # the tilings a later autotune may pick: the plain and stacked bn = 64 operands, streamed for per-image weights
    assert {(64, (1, 1)), (64, (1, 9)), (128, (1, 1))} <= cfgs_seen["swish"], cfgs_seen["swish"]
    assert {(64, (1, 5)), (64, (1, 13)), (128, (1, 5))} <= cfgs_seen["per-image"], cfgs_seen["per-image"]
