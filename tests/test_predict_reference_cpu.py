"""CPU: the float64 reference of the prediction stage's kernels (tests/predict_reference.py) against PyTorch's own
definitions of the same operations in float64 (F.layer_norm, F.gelu, torch.sigmoid, torch.softmax, a depthwise
F.conv2d, F.pad + F.max_pool2d), every magnitude it states bounding |value|, and a guard that every launch of the eight
entry points goes through the dense wrapper tests/test_predict_contract_gpu.py records."""
import ast
import os

import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import dense
from tests import predict_reference as R

F64 = torch.float64


def _rand(*shape, seed, scale=1.0, offset=0.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=F64) * scale + offset


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    assert float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-300), float((a - b).abs().max())


def _bounds(r):
    assert bool((r["mag"] >= r["y"].abs() * (1 - 1e-12)).all()), "a magnitude below |value|"


def _ln_params(C, seed):
    return _rand(C, seed=seed).float(), _rand(C, seed=seed + 1, scale=0.5).float(), 1e-6


# ------------------------------------------------------------------------------------------------ GRU
def test_gru_gates_and_update():
    r, u = _rand(3, 5, 7, 64, seed=1, scale=6.0), _rand(3, 5, 7, 64, seed=2, scale=6.0)
    h, ht = _rand(3, 5, 7, 64, seed=3), _rand(3, 5, 7, 64, seed=4)
    g = R.gru_gates(r, h)
    _close(g["y"], (1 - torch.sigmoid(r)) * h)
    _bounds(g)
    up = R.gru_update(u, h, ht)
    s = torch.sigmoid(u)
    _close(up["y"], h + s * (ht - h))
    _bounds(up)


def test_saturated_gates_are_the_limits():
    big = torch.tensor([-200.0, -60.0, 60.0, 200.0], dtype=F64)
    h, ht = torch.full((4,), 3.0, dtype=F64), torch.full((4,), -5.0, dtype=F64)
    _close(R.gru_gates(big, h)["y"], torch.tensor([3.0, 3.0, 0.0, 0.0], dtype=F64), tol=1e-15)
    _close(R.gru_update(big, h, ht)["y"], torch.tensor([3.0, 3.0, -5.0, -5.0], dtype=F64), tol=1e-15)


def test_gru_and_mix_compose_to_the_oracles_dual_gru():
    """gru_gates, gru_update and trust_mix, wired as the sm_90a Dual_GRU wires them (gates raw out of the convolutions),
    reproduce one future step of oracle/torch_predict.py's dual_gru, which tests/test_predict_oracle_cpu.py pins to the
    reference's own FuturePrediction: the gate roles ((1 - r) h, (1 - u) h + u h_tilde) and which softmax output weighs
    which state (p0 s2 + p1 s1) are the reference's, not restatements of the same expressions"""
    from oracle import torch_predict as TP
    from stp3_b200.layers.temporal import Dual_GRU
    from stp3_b200.utils import synthetic as syn
    m = Dual_GRU(32, 64, n_future=1)
    syn.init_exact(m, seed=3)
    m = m.double().eval()
    H, W = 5, 6
    x, state = _rand(1, 1, 32, H, W, seed=70), _rand(1, 2, 64, H, W, seed=71)
    cl = lambda t: t.permute(0, 2, 3, 1)           # noqa: E731
    cf = lambda t: t.permute(0, 3, 1, 2)           # noqa: E731

    def cell(a, h, cu, cr, ct):
        xh = torch.cat([a, h], 1)
        g = cf(R.gru_gates(cl(TP._conv(xh, cr)), cl(h))["y"])
        ht = TP._conv(torch.cat([a, g], 1), ct)
        return cf(R.gru_update(cl(TP._conv(xh, cu)), cl(h), cl(ht))["y"])
    with torch.no_grad():
        ref = TP.dual_gru(x, state, m)[:, 0]
        h = cell(state[:, 0], state[:, 0], m.conv_update_2, m.conv_reset_2, m.conv_state_tilde_2)
        s1 = cell(x[:, 0], state[:, 1], m.conv_update_1, m.conv_reset_1, m.conv_state_tilde_1)
        h = cell(state[:, 1], h, m.conv_update_2, m.conv_reset_2, m.conv_state_tilde_2)
        s2 = TP._conv(h, m.conv_decoder_2)
        t = TP.bottleblock(torch.cat([s1, s2], 1), m.trusting_gate[0])
        w = m.trusting_gate[1].weight.reshape(2, 64)
        got = cf(R.trust_mix(cl(t), w, cl(s1), cl(s2))["y"])
    _close(got, ref)
    swapped = cf(R.trust_mix(cl(t), w, cl(s2), cl(s1))["y"])
    assert float((swapped - ref).abs().max()) > 1e-3 * float(ref.abs().max())     # the check sees the order


# ------------------------------------------------------------------------------------------------ LayerNorm / GELU
@pytest.mark.parametrize("C", [8, 16, 24, 32, 64, 136, 200, 256])
def test_channel_norm_act_matches_layer_norm_and_gelu(C):
    x = _rand(2, 3, 5, C, seed=C)
    g, b, eps = _ln_params(C, 10 + C)
    ref = F.layer_norm(x, (C,), g.double(), b.double(), R.f32(eps))
    r = R.channel_norm_act(x, (g, b, eps))
    _close(r["y"], ref)
    _bounds(r)
    y = _rand(2, 3, 5, C, seed=20 + C)
    for gelu_y in (False, True):
        r = R.channel_norm_act(x, (g, b, eps), act=True, y=y, gelu_y=gelu_y)
        _close(r["y"], F.gelu(ref) + (F.gelu(y) if gelu_y else y))
        _bounds(r)
    r = R.channel_norm_act(x, act=True)
    _close(r["y"], F.gelu(x))
    _bounds(r)


def test_layer_norm_at_a_large_mean():
    """mean 1e3, spread 1e-2: the reference normalises the spread, which a one-pass E[x^2] - E[x]^2 in fp32 loses"""
    x = _rand(4, 64, seed=5, scale=1e-2, offset=1e3)
    g, b, eps = _ln_params(64, 6)
    r = R.channel_norm_act(x, (g, b, eps))
    _close(r["y"], F.layer_norm(x, (64,), g.double(), b.double(), R.f32(eps)), tol=1e-9)
    _bounds(r)
    one_pass = (x.float() ** 2).mean(-1) - x.float().mean(-1) ** 2
    assert float((one_pass.double() - x.var(-1, unbiased=False)).abs().max()) > 10 * float(x.var(-1).max())


# ------------------------------------------------------------------------------------------------ depthwise + LN
@pytest.mark.parametrize("k, H, W", [(7, 9, 11), (1, 4, 5), (3, 1, 1), (15, 1, 6), (15, 6, 1), (3, 5, 1), (7, 2, 3)])
def test_dw_ln_matches_depthwise_conv2d_and_layer_norm(k, H, W):
    C = 24
    x = _rand(2, H, W, C, seed=k + H)
    w, b = _rand(k * k, C, seed=30 + k).float(), _rand(C, seed=40 + k).float()
    g, beta, eps = _ln_params(C, 50)
    wc = w.double().t().reshape(C, 1, k, k)
    a = F.conv2d(x.permute(0, 3, 1, 2), wc, b.double(), padding=k // 2, groups=C).permute(0, 2, 3, 1)
    r = R.dw_ln(x, w, b, k, g, beta, eps)
    _close(r["y"], F.layer_norm(a, (C,), g.double(), beta.double(), R.f32(eps)))
    _bounds(r)
    acc, mag = R.depthwise(x, w, b, k)
    _close(acc, a)
    amag = F.conv2d(x.abs().permute(0, 3, 1, 2), wc.abs(), b.double().abs(), padding=k // 2, groups=C).permute(0, 2, 3, 1)
    _close(mag, amag)


# ------------------------------------------------------------------------------------------------ trusting gate
@pytest.mark.parametrize("scale", [1.0, 100.0])
def test_trust_mix_matches_softmax(scale):
    """logits up to ~1e3 apart (scale 100): the softmax stays finite and saturates"""
    C = 64
    t, w = _rand(3, 4, C, seed=60, scale=scale), _rand(2, C, seed=61).float()
    s1, s2 = _rand(3, 4, C, seed=62), _rand(3, 4, C, seed=63)
    p = torch.softmax(t @ w.double().t(), -1)
    r = R.trust_mix(t, w, s1, s2)
    _close(r["y"], s2 * p[..., :1] + s1 * p[..., 1:])
    assert bool(torch.isfinite(r["y"]).all())
    _bounds(r)


# ------------------------------------------------------------------------------------------------ pad + max pool
@pytest.mark.parametrize("H, W", [(13, 13), (25, 25), (1, 7), (6, 1), (1, 1), (4, 6)])
def test_maxpool2_pad_matches_pad_and_max_pool2d(H, W):
    x = _rand(2, H, W, 16, seed=H * 100 + W).float()
    hi, lo = R.split(x)
    v = R.planes(hi, lo).permute(0, 3, 1, 2)
    ref = F.max_pool2d(F.pad(v, (0, W % 2, 0, H % 2)), 2, 2).permute(0, 2, 3, 1)
    oh, ol = R.maxpool2_pad(hi, lo)
    assert torch.equal(R.planes(oh, ol), ref)
    # every output pair is one of its window's stored pairs, or the +0 / +0 of the padding
    assert not bool(oh.isnan().any())


def test_maxpool2_pad_keeps_the_first_of_equal_values():
    """-0 before +0 keeps -0's bits; a padded +0 never replaces a -0 before it"""
    hi = torch.tensor([-0.0, 0.0, 0.0, -0.0, -0.0], dtype=torch.float32).to(torch.bfloat16).view(1, 1, 5, 1)
    hi = hi.expand(1, 1, 5, 8).contiguous()
    lo = torch.zeros_like(hi)
    oh, _ = R.maxpool2_pad(hi, lo)
    bits = oh.contiguous().view(torch.int16)[0, 0, :, 0].tolist()
    assert bits == [-32768, 0, -32768], bits


# ------------------------------------------------------------------------------------------------ recorder guard
# entry point -> the dense function that wraps it (tests/test_predict_contract_gpu.py records these functions)
WRAPPERS = {"stp3_gru_gates": "gru_gates", "stp3_gru_update": "gru_update", "stp3_channel_norm_act": "channel_norm_act",
            "stp3_dw_ln": "dw_ln", "stp3_trust_mix": "trust_mix", "stp3_maxpool2_pad": "maxpool2_pad",
            "stp3_hl_copy": "hl_copy", "stp3_hl_broadcast": "hl_broadcast"}


def predict_calls_outside_the_wrappers():
    """Uses of the eight entry points anywhere in the package except inside their dense.py wrapper, imports of a wrapper
    by name, and calls of a wrapper by its bare name: each would launch a kernel the recorder, which replaces the dense
    module's attributes, may not see."""
    pkg = os.path.dirname(os.path.abspath(dense.__file__))
    allowed = {(os.path.abspath(dense.__file__), fn, sym) for sym, fn in WRAPPERS.items()}
    wrappers = set(WRAPPERS.values())
    bad = []
    for root, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            path = os.path.join(root, f)
            with open(path) as fh:
                tree = ast.parse(fh.read())
            owner = {}
            for fn in ast.walk(tree):
                if isinstance(fn, (ast.FunctionDef, ast.AsyncFunctionDef)):
                    for n in ast.walk(fn):
                        owner.setdefault(id(n), fn.name)     # the outermost function wins (ast.walk is breadth first)
            for n in ast.walk(tree):
                if isinstance(n, ast.ImportFrom) and any(a.name in wrappers for a in n.names):
                    bad.append(f"{f}:{n.lineno} imports {[a.name for a in n.names]}")
                elif isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id in wrappers:
                    bad.append(f"{f}:{n.lineno} calls {n.func.id} by its bare name")
                elif isinstance(n, ast.Attribute) and n.attr in WRAPPERS:
                    if (path, owner.get(id(n)), n.attr) not in allowed:
                        bad.append(f"{f}:{n.lineno} {n.attr} in {owner.get(id(n))}")
    return bad


def test_every_call_goes_through_a_recorded_wrapper():
    assert not predict_calls_outside_the_wrappers()
