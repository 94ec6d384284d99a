"""CPU: the fp64 prediction-stage oracle (oracle/torch_predict.py) against what the unmodified reference computed
(tests/golden/predict_*.npz, oracle/make_golden_predict.py), the refusals of the Prediction configurations, the
reference's parameter names, and the Bottleneck skip's pad-then-maxpool rule."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import torch_predict as TP
from oracle.make_golden_predict import _Stage, module_states, predict_cfg, predict_modules
from stp3_b200.config import PREDICTION_OVERRIDES, get_cfg
from stp3_b200.models.stp3 import STP3

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    return np.load(os.path.join(GOLD, f"predict_{name}.npz"))


def check_key(g, key, got64):
    """The oracle reproduces its own stored values and sits within 1e-4 of max of the reference's fp32 values."""
    idx = g[f"{key}_index"]
    got = got64.reshape(-1)[torch.from_numpy(idx.astype(np.int64))].numpy()
    mx = float(g[f"{key}_max"])
    assert tuple(got64.shape) == tuple(g[f"{key}_shape"])
    assert np.abs(got - g[f"{key}_oracle"]).max() <= 1e-10 * mx, key
    dev = np.abs(got - g[f"{key}_ref"].astype(np.float64)).max() / mx
    assert dev < 1e-4, (key, dev)


@pytest.mark.parametrize("probabilistic", [True, False])
def test_oracle_matches_reference_modules_48x64(probabilistic):
    g = golden("modules_48x64" if probabilistic else "noprob_48x64")
    mods = copy.deepcopy(predict_modules(probabilistic=probabilistic)).double()
    states = module_states().double()
    with torch.no_grad():
        if probabilistic:
            mls = TP.distribution(states[:, -1:], mods.present_distribution)
            check_key(g, "mu_log_sigma", mls)
            x = mls[:, :, :32].view(2, 1, 32, 1, 1).expand(2, 1, 32, 48, 64)
            check_key(g, "dual_gru", TP.dual_gru(x, states, mods.future_prediction.dual_grus))
        check_key(g, "future", TP.predict_stage(states, _Stage(mods, probabilistic)))


@pytest.mark.parametrize("name", ["e2e_nuscenes", "e2e_carla"])
def test_end_to_end_fixtures(name):
    """The 200 x 200 fixtures the GPU test compares against.  The present states (the temporal model's output) and the
    present-frame hdmap of the reference's fp32 run sit within 1e-4 of max of the fp64 oracle.  Through the
    recurrences the synthetic weights amplify every rounding (DESIGN.md §3.16): the fixture records the reference's
    own full-tensor distance from fp64 (`fulldev`), and every stored sample lies within it."""
    g = golden(name)
    keys = sorted({k[:-len("_max")] for k in g.files if k.endswith("_max")})
    heads = {"e2e_nuscenes": {"segmentation", "instance_center", "instance_offset", "instance_flow"},
             "e2e_carla": {"segmentation", "pedestrian", "hdmap"}}[name]
    assert set(keys) == {"states", "future"} | heads
    assert tuple(g["future_shape"]) == (1, 7, 64, 200, 200) and tuple(g["states_shape"]) == (1, 3, 64, 200, 200)
    for key in keys:
        dev = np.abs(g[f"{key}_ref"].astype(np.float64) - g[f"{key}_oracle"]).max() / float(g[f"{key}_max"])
        assert np.isfinite(g[f"{key}_fulldev"]) and dev <= float(g[f"{key}_fulldev"]), key
        if key in ("states", "hdmap"):
            assert dev < 1e-4, (key, dev)


def test_maxpool_pads_odd_edges_with_zeros():
    """F.pad(value=0) precedes the pool: the padded zeros take part in the max of the last row / column."""
    x = -torch.arange(1, 1 + 2 * 3 * 5, dtype=torch.float64).view(1, 2, 3, 5)
    y = TP.maxpool2_pad(x)
    assert y.shape == (1, 2, 2, 3)
    assert torch.equal(y[0, 0, 0, :2], torch.tensor([-1.0, -3.0], dtype=torch.float64))
    assert (y[0, :, 1, :] == 0).all() and (y[0, :, :, 2] == 0).all()
    x = torch.randn(2, 3, 25, 13, dtype=torch.float64).abs() + 1
    y = TP.maxpool2_pad(x)
    assert y.shape == (2, 3, 13, 7)
    assert torch.equal(y[:, :, :12, :6], torch.nn.functional.max_pool2d(x[:, :, :24, :12], 2))
    assert torch.equal(y[:, :, 12, :6], torch.maximum(x[:, :, 24, 0:12:2], x[:, :, 24, 1:12:2]))


def test_parameter_names_match_the_reference():
    """The Prediction model's present_distribution / future_prediction state dict has the reference's keys and shapes
    (recorded from the reference modules), so a Prediction checkpoint loads with strict=True."""
    g = golden("modules_48x64")
    ref = dict(zip(g["ref_keys"].tolist(), g["ref_key_shapes"].tolist()))
    for carla in (False, True):
        model = STP3(predict_cfg(carla), backbone=torch.nn.Identity())
        ours = {k: str(tuple(v.shape)) for k, v in model.state_dict().items()
                if k.startswith(("present_distribution.", "future_prediction."))}
        assert ours == ref
    sd = model.state_dict()
    STP3(predict_cfg(True), backbone=torch.nn.Identity()).load_state_dict(sd, strict=True)


def test_reference_state_dict_loads_strict_when_available():
    from oracle.ref_loader import load_reference, reference_available
    if not reference_available():
        pytest.skip("the reference is not installed under oracle/_ref/")
    ref = load_reference()
    import stp3.models.distributions as RD
    import stp3.models.future_prediction as RF
    for carla in (False, True):
        cfg = predict_cfg(carla)
        model = STP3(cfg, backbone=torch.nn.Identity())
        sd = dict(model.state_dict())
        parts = {"present_distribution": RD.DistributionModule(64, 32, method="GAUSSIAN"),
                 "future_prediction": RF.FuturePrediction(64, 32, 4),
                 "decoder": ref.decoder.Decoder(64, 2, 3, 2, dict(
                     perceive_hdmap=cfg.SEMANTIC_SEG.HDMAP.ENABLED,
                     predict_pedestrian=cfg.SEMANTIC_SEG.PEDESTRIAN.ENABLED, predict_instance=cfg.INSTANCE_SEG.ENABLED,
                     predict_future_flow=cfg.INSTANCE_FLOW.ENABLED, planning=False))}
        for pre, m in parts.items():
            torch.manual_seed(0)
            for p in m.state_dict().values():
                if p.is_floating_point():
                    p.copy_(torch.randn_like(p))
            for k, v in m.state_dict().items():
                sd[f"{pre}.{k}"] = v
        model.load_state_dict(sd, strict=True)
        assert torch.equal(model.future_prediction.dual_grus.conv_update_1.weight,
                           parts["future_prediction"].dual_grus.conv_update_1.weight)


def _cfg(**over):
    cfg = get_cfg(PREDICTION_OVERRIDES, perception=False)
    return cfg.merge(over)


@pytest.mark.parametrize("over, needle", [
    ({"PROBABILISTIC": {"METHOD": "BERNOULLI"}}, "BERNOULLI"),
    ({"PROBABILISTIC": {"METHOD": "MIXGAUSSIAN"}}, "MIXGAUSSIAN"),
    ({"PLANNING": {"ENABLED": True}}, "PLANNING"),
    ({"MODEL": {"TEMPORAL_MODEL": {"NAME": "identity"}}}, "identity temporal model"),
])
def test_unsupported_prediction_configs_are_refused(over, needle):
    with pytest.raises(NotImplementedError, match=needle):
        STP3(_cfg(**over), backbone=torch.nn.Identity())


def test_prediction_without_probabilistic_builds_no_distribution():
    model = STP3(_cfg(PROBABILISTIC={"ENABLED": False}), backbone=torch.nn.Identity())
    assert not hasattr(model, "present_distribution") and hasattr(model, "future_prediction")


def _inputs():
    B, S, N, C, D, Hf, Wf = 1, 3, 6, 64, 48, 28, 60
    return (torch.zeros(B, S, N, C, Hf, Wf), torch.zeros(B, S, N, D, Hf, Wf), torch.eye(3).expand(B, S, N, 3, 3),
            torch.eye(4).expand(B, S, N, 4, 4), torch.zeros(B, S, 6))


@pytest.mark.parametrize("where", ["model", "future_prediction", "present_distribution", "block"])
def test_train_mode_is_refused_as_eval_only(where):
    model = STP3(_cfg(), backbone=torch.nn.Identity()).eval()
    target = {"model": model, "future_prediction": model.future_prediction,
              "present_distribution": model.present_distribution,
              "block": model.future_prediction.res_blocks1[0]}[where]
    target.train()
    with pytest.raises(NotImplementedError, match="prediction stage .* is eval-only"):
        model.forward_features(*_inputs())


@pytest.mark.parametrize("entry", ["forward", "forward_trunk_features", "forward_heads_device", "native_forward",
                                   "forward_images_device"])
def test_every_entry_point_refuses_train_mode_first(entry):
    """A train-mode Prediction model is refused with the eval-only message before any trunk, head or lift-splat work,
    whichever entry point it is called through (the native trunk's own train-mode checks would otherwise fire
    first)."""
    native = entry in ("native_forward", "forward_images_device")
    if native:
        from stp3_b200.models.efficientnet import EfficientNetTrunk
        model = STP3(_cfg(), backbone=EfficientNetTrunk("b0", trainable=True))
    else:
        model = STP3(_cfg(), backbone=torch.nn.Identity())
    model.train()
    feat, depth, intr, extr, ego = _inputs()
    image = torch.zeros(1, 3, 6, 3, 224, 480)
    r_lo, r_hi = torch.zeros(1, 3, 6, 112, 28, 60), torch.zeros(1, 3, 6, 160, 14, 30)
    host = (torch.zeros(1, 3, 6, 3, 3), torch.zeros(1, 3, 6, 3), torch.zeros(1, 3, 3, 3), torch.zeros(1, 3, 3),
            torch.zeros(3, 6))
    call = {"forward": lambda: model(image, intr, extr, ego),
            "native_forward": lambda: model(image, intr, extr, ego),
            "forward_trunk_features": lambda: model.forward_trunk_features(r_lo, r_hi, intr, extr, ego),
            "forward_heads_device": lambda: model.forward_heads_device(r_lo, r_hi, *host),
            "forward_images_device": lambda: model.forward_images_device(image, *host)}[entry]
    with pytest.raises(NotImplementedError, match="prediction stage .* is eval-only"):
        call()


def test_layer_norm_refuses_train_mode():
    from stp3_b200.layers.convolutions import LayerNorm
    with pytest.raises(NotImplementedError, match="eval-only"):
        LayerNorm(64)(torch.zeros(2, 4, 4, 64))


def test_module_forward_refuses_train_mode():
    model = STP3(_cfg(), backbone=torch.nn.Identity())
    for m in (model.future_prediction.dual_grus, model.future_prediction.spatial_grus[0],
              model.future_prediction.res_blocks1[0], model.future_prediction.dual_grus.trusting_gate[0],
              model.present_distribution.encoder.model[0]):
        m.train()
        with pytest.raises(NotImplementedError, match="eval-only"):
            m.forward_hl(None, None, None) if m is model.future_prediction.dual_grus else \
                m.forward_hl(None, None) if m is model.future_prediction.spatial_grus[0] else m.forward_hl(None)


def test_frame_sharded_mode_is_refused_with_prediction():
    model = STP3(_cfg(), backbone=torch.nn.Identity()).eval()
    feat, depth, intr, extr, ego = _inputs()
    with pytest.raises(NotImplementedError, match="frame-sharded .* N_FUTURE_FRAMES"):
        model.forward_features_frame_sharded(feat, depth, intr, extr, ego)


def test_perception_config_is_unchanged():
    """N_FUTURE_FRAMES = 0 builds no prediction module: the perception state dict keeps its keys."""
    model = STP3(get_cfg(), backbone=torch.nn.Identity())
    assert not any(k.startswith(("present_distribution", "future_prediction")) for k in model.state_dict())
