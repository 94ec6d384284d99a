"""CPU: the train-mode DeepLab head's oracle, its dilated input-gradient tables and the argument checks of the changed
C entry points.

(a) The fp64 train-mode restatement (oracle/torch_deeplab_train.deeplab_head_train) against tests/golden/deeplab_train_*.npz,
    which the reference's own DeepLabHead produced in train mode with a fixed dropout mask
    (oracle/make_golden_head_train.py): output and running statistics to 1e-5, every gradient and the input gradient to
    1e-4 of the tensor's max, with the ReLU branches pinned to the reference's where an input lies within round-off of
    zero (stored in the fixture).
(b) The dilated input-gradient tap tables (dense_train.dgrad_taps, e = pad - k * d), evaluated in fp64 with F.conv2d,
    reproduce torch.nn.grad.conv2d_input.
(c) stp3_conv_wgrad refuses dilation < 1 and stp3_bn_apply a dropout p outside [0, 1), before touching memory."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_dense as TD
from oracle import torch_dense_train as TT
from oracle import torch_deeplab_train as TH
from stp3_b200 import _lib
from stp3_b200 import dense_train as T
from stp3_b200.layers.convolutions import DeepLabHead


@pytest.mark.parametrize("name", ["temporal", "encoder"])
def test_fp64_train_oracle_matches_reference_fixture(name):
    golden = np.load(f"tests/golden/deeplab_train_{name}.npz")
    cin, ncls, hidden = (int(v) for v in golden["cfg"])
    N, _, H, W = (int(v) for v in golden["shape"])
    head = TD.init_exact(DeepLabHead(cin, ncls, hidden_channel=hidden), seed=3)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = float(golden["momentum"])
    head = head.double().train()
    x = TD.exact_gauss((N, cin, H, W), torch.Generator().manual_seed(5)).double().requires_grad_(True)
    mask = TH.dropout_keep_mask((N, hidden, H, W), int(golden["mask_seed"]), float(golden["p"]))
    calls = []

    def relu(t):
        k = len(calls)
        calls.append(k)
        m = (t.detach() > 0).reshape(-1)
        idx = torch.from_numpy(golden[f"relu{k}_idx"].astype(np.int64))
        m[idx] = torch.from_numpy(golden[f"relu{k}_pos"])
        return t * m.view(t.shape).to(t.dtype)
    out = TH.deeplab_head_train(x, head, relu=relu, dropout_mask=mask)
    assert len(calls) == int(golden["n_relu"])
    G = TT.upstream_grads({"out": out}, seed=9)["out"]
    (out * G.double()).sum().backward()
    flat = out.detach().reshape(-1)
    s = golden["out_s"]
    e = np.abs(flat[TT.sample_index("out", flat.numel(), len(s))].numpy() - s).max() / golden["out_amax"]
    assert e < 1e-5, e
    for k, b in head.named_buffers():
        want = golden[k]
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(want), k
            continue
        e = np.abs(b.numpy() - want).max() / np.abs(want).max()
        assert e < 1e-5, (k, e)
    for k, p in list(head.named_parameters()) + [("x", x)]:
        flat = p.grad.reshape(-1)
        s = golden[f"grad_{k}_s"]
        e = np.abs(flat[TT.sample_index(f"grad.{k}", flat.numel(), len(s))].numpy() - s).max() / golden[f"grad_{k}_amax"]
        assert e < 1e-4, (k, e)


@pytest.mark.parametrize("hw", [(14, 30), (25, 25)])
@pytest.mark.parametrize("d", [1, 12, 24, 36])
def test_dilated_dgrad_tap_tables_reproduce_conv2d_input(d, hw):
    H, W = hw
    gen = torch.Generator().manual_seed(d)
    cin, cout, N = 5, 6, 2
    w = torch.randn((cout, cin, 3, 3), generator=gen, dtype=torch.float64)
    g = torch.randn((N, cout, H, W), generator=gen, dtype=torch.float64)
    ref = torch.nn.grad.conv2d_input((N, cin, H, W), w, g, padding=d, dilation=d)
    (ph, taps), = T.dgrad_taps(3, 3, 1, d, d)
    assert ph == (0, 0) and len(taps) == 9
    P = max(max(abs(ey), abs(ex)) for _, _, ey, ex in taps)
    gp = F.pad(g, (P, P, P, P))
    got = torch.zeros_like(ref)
    for ky, kx, ey, ex in taps:
        win = gp[:, :, P + ey:P + ey + H, P + ex:P + ex + W]                 # g[i + ey, j + ex], zero outside
        got += F.conv2d(win, w[:, :, ky, kx].t().reshape(cin, cout, 1, 1))
    e = ((got - ref).abs().max() / ref.abs().max()).item()
    assert e < 1e-12, e


def test_dgrad_taps_refuse_bad_dilation():
    with pytest.raises(ValueError, match="dilation"):
        T.dgrad_taps(3, 3, 1, 1, 0)
    with pytest.raises(NotImplementedError, match="dilated stride-2"):
        T.dgrad_taps(3, 3, 2, 2, 2)


FAKE = 1 << 20   # a non-null, aligned device address: every call below is refused before it is dereferenced


def test_changed_entry_points_refuse_bad_arguments():
    if not __import__("os").path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    assert L.stp3_abi_version() == 7
    assert L.stp3_conv_wgrad_scratch_bytes(2, 14, 30, 64, 160, 3, 3, 0) == 0
    assert L.stp3_conv_wgrad_scratch_bytes(2, 14, 30, 64, 160, 3, 3, 36) == \
        L.stp3_conv_wgrad_scratch_bytes(2, 14, 30, 64, 160, 3, 3, 1) > 0
    for dil in (0, -1):
        rc = L.stp3_conv_wgrad(FAKE, 2, 14, 30, 160, 160, FAKE, 14, 30, 64, 64, 3, 3, 1, 1, dil, FAKE, 1 << 40, FAKE, None)
        assert rc == -1 and b"dilation must be >= 1" in L.stp3_last_error(), dil
    for p in (1.0, 1.5, -0.1, float("nan")):
        rc = L.stp3_bn_apply(FAKE, 100, 64, 64, FAKE, FAKE, FAKE, FAKE, None, 0, 1, p, 1, 0, FAKE, 64, None, None, 0, None)
        assert rc == -1 and b"dropout p must be in [0, 1)" in L.stp3_last_error(), p
    rc = L.stp3_image_channel_sums(FAKE, 2, 100, 64, 64, FAKE, FAKE, 0, None)
    assert rc == -1 and b"scratch smaller" in L.stp3_last_error()
