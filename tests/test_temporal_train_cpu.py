"""CPU: the host pieces of the train-mode TemporalBlocks -- the anti-causal input-gradient tap tables of the causal 3-D
convolutions and the pyramid-pooling pair mean with its adjoint, in fp64 -- the train-mode restatement
(oracle/torch_temporal_train) against tests/golden/temporal_train_*.npz, which the reference's own TemporalModel produced
in train mode with a fixed head dropout mask (oracle/make_golden_temporal_train.py), and against reference-shaped
modules, and the new entry points' argument refusals."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_dense as TD
from oracle import torch_dense_train as TT
from oracle import torch_deeplab_train as TH
from oracle import torch_temporal_train as OT
from stp3_b200 import _lib, dense_train as T
from stp3_b200.layers.temporal import TemporalBlock
from stp3_b200.models.temporal_model import TemporalModel


@pytest.mark.parametrize("name", ["perceive", "stress"])
def test_fp64_train_oracle_matches_reference_fixture(name):
    """Output and running statistics to 1e-5, every gradient (input included) to 1e-4 of the tensor's max, with the
    ReLU branches pinned to the reference's where an input lies within round-off of zero (stored in the fixture)."""
    golden = np.load(f"tests/golden/temporal_train_{name}.npz")
    B, S, cin, H, W = (int(v) for v in golden["shape"])
    tm = TD.init_exact(TemporalModel(cin, S, (H, W), start_out_channels=64), seed=3)
    for m in tm.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = float(golden["momentum"])
    tm = tm.double().train()
    x = TD.exact_gauss((B, S, cin, H, W), torch.Generator().manual_seed(5)).double().requires_grad_(True)
    mask = TH.dropout_keep_mask((B * S, int(golden["hidden"]), H, W), int(golden["mask_seed"]), float(golden["p"]))
    calls = []

    def relu(t):
        k = len(calls)
        calls.append(k)
        m = (t.detach() > 0).reshape(-1)
        idx = torch.from_numpy(golden[f"relu{k}_idx"].astype(np.int64))
        m[idx] = torch.from_numpy(golden[f"relu{k}_pos"])
        return t * m.view(t.shape).to(t.dtype)
    out = OT.temporal_model_train(x, tm, relu=relu, dropout_mask=mask)
    assert len(calls) == int(golden["n_relu"])
    G = TT.upstream_grads({"out": out}, seed=9)["out"].double()
    (out * G).sum().backward()
    flat = out.detach().reshape(-1)
    e = np.abs(flat[TT.sample_index("out", flat.numel(), len(golden["out_s"]))].numpy() - golden["out_s"]).max()
    assert e / golden["out_amax"] < 1e-5, e
    for k, b in tm.named_buffers():
        ref = golden[k]
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(ref) == 1, k
            continue
        e = np.abs(b.numpy() - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert e < 1e-5, (k, e)
    worst = 0.0
    for k, p in list(tm.named_parameters()) + [("x", x)]:
        flat = p.grad.reshape(-1)
        s = golden[f"grad_{k}_s"]
        e = np.abs(flat[TT.sample_index(f"grad.{k}", flat.numel(), len(s))].numpy() - s).max() / golden[f"grad_{k}_amax"]
        worst = max(worst, e)
        assert e < 1e-4, (k, e)
    print(f"{name}: worst gradient {worst:.2e} of max")


def causal_conv3d(x, w):
    kt, kh, kw = w.shape[2:]
    return F.conv3d(F.pad(x, ((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0)), w)


@pytest.mark.parametrize("k", [(2, 3, 3), (1, 3, 3), (1, 1, 1), (3, 3, 3)])
@pytest.mark.parametrize("t", [1, 2, 5])
def test_anticausal_dgrad_tap_tables_reproduce_conv3d_input(k, t):
    gen = torch.Generator().manual_seed(t)
    cin, cout, B, H, W = 5, 6, 2, 7, 9
    x = torch.randn((B, cin, t, H, W), generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn((cout, cin, *k), generator=gen, dtype=torch.float64)
    g = torch.randn((B, cout, t, H, W), generator=gen, dtype=torch.float64)
    (ref,) = torch.autograd.grad(causal_conv3d(x, w), x, g)
    taps = T.dgrad_taps_3d(*k)
    assert len(taps) == k[0] * k[1] * k[2] and all(et >= 0 for _, _, _, et, _, _ in taps)
    P = max(max(abs(ey), abs(ex), et) for _, _, _, et, ey, ex in taps)
    gp = F.pad(g, (P, P, P, P, P, P))
    got = torch.zeros_like(ref)
    for it, ky, kx, et, ey, ex in taps:
        win = gp[:, :, P + et:P + et + t, P + ey:P + ey + H, P + ex:P + ex + W]   # g[t + et, i + ey, j + ex], zero outside
        got += F.conv3d(win, w[:, :, it, ky, kx].t().reshape(cin, cout, 1, 1, 1))
    e = ((got - ref).abs().max() / ref.abs().max()).item()
    assert e < 1e-12, e


def test_dgrad_taps_3d_refuse_non_square_kernels():
    for k in ((2, 3, 1), (2, 2, 2)):
        with pytest.raises(ValueError, match="square and odd"):
            T.dgrad_taps_3d(*k)


@pytest.mark.parametrize("t", [2, 3, 5])
def test_pair_mean_is_the_reference_avgpool_and_its_adjoint(t):
    gen = torch.Generator().manual_seed(t)
    B, C, H, W = 2, 7, 3, 4
    x = torch.randn((B, C, t, H, W), generator=gen, dtype=torch.float64)
    pool = torch.nn.AvgPool3d((2, H, W), stride=(1, H, W), padding=(1, 0, 0), count_include_pad=False)
    ref = pool(x).reshape(B, C, t + 1).permute(0, 2, 1).reshape(B * (t + 1), C)
    m = x.mean(dim=(3, 4)).permute(0, 2, 1).reshape(B * t, C)
    assert (OT.pair_mean(m, t) - ref).abs().max() < 1e-14
    # the adjoint of stp3_temporal_pair_mean: c_t g[t] + g[t+1] / 2 (t + 1 < T), c_t g[t] + g[T] (t = T - 1)
    g = torch.randn((B * (t + 1), C), generator=gen, dtype=torch.float64)
    gt = g.view(B, t + 1, C)
    adj = gt[:, :t].clone()
    adj[:, 1:] *= 0.5
    adj[:, :-1] += 0.5 * gt[:, 1:t]
    adj[:, -1] += gt[:, t]
    mm = m.clone().requires_grad_(True)
    (auto,) = torch.autograd.grad(OT.pair_mean(mm, t), mm, g)
    assert (adj.view(B * t, C) - auto).abs().max() < 1e-14


def test_restatement_matches_reference_modules():
    """The restatement's block against the same block run through nn modules shaped like the reference's forward
    (pad, Conv3d, BatchNorm3d in train mode, AvgPool3d, bilinear upsampling)."""
    torch.manual_seed(0)
    blk = TemporalBlock(70, 64, use_pyramid_pooling=True, pool_sizes=[(2, 6, 8)]).double().train()
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            with torch.no_grad():
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    x = torch.randn((2, 70, 3, 6, 8), dtype=torch.float64)
    ref_blk = copy.deepcopy(blk)
    got = OT.temporal_block_train(x, blk)
    paths = []
    for i, path in enumerate(ref_blk.convolution_paths):
        e = path[0] if i < 2 else path
        y = F.relu(e.norm(e.conv(x)))
        if i < 2:
            cc = path[1]
            y = F.relu(cc.norm(cc.conv(cc.pad(y))))
        paths.append(y)
    pp = ref_blk.pyramid_pooling.features[0]
    v = pp.conv_bn_relu(pp.avgpool(x))[:, :, :-1]
    b, c, t = v.shape[:3]
    v = F.interpolate(v.permute(0, 2, 1, 3, 4).reshape(b * t, c, 1, 1), (6, 8), mode="bilinear",
                      align_corners=False).view(b, t, c, 6, 8).permute(0, 2, 1, 3, 4)
    r = ref_blk.aggregation(torch.cat(paths + [v], 1))
    want = ref_blk.projection(x) + r
    assert (got - want).abs().max() < 1e-10
    for (k, a), (_, b_) in zip(blk.named_buffers(), ref_blk.named_buffers()):
        assert torch.allclose(a.double(), b_.double(), atol=1e-12), k


FAKE = 1 << 20   # a non-null, aligned device address: every call below is refused before it is dereferenced


def test_new_entry_points_refuse_bad_arguments():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    assert L.stp3_abi_version() == 7
    assert L.stp3_conv3d_wgrad_scratch_bytes(2, 3, 48, 64, 35, 35, 2, 3, 3) > 0
    assert L.stp3_conv3d_wgrad_scratch_bytes(2, 0, 48, 64, 35, 35, 2, 3, 3) == 0
    ok = (FAKE, 2, 3, 48, 64, 35, 35, FAKE, 35, 35, 2, 3, 3, FAKE, 1 << 40, FAKE, None)

    def call(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return L.stp3_conv3d_wgrad(*a), L.stp3_last_error()
    for kw, msg in [({"a0": None}, b"null pointer"), ({"a15": None}, b"null pointer"),
                    ({"a2": 0}, b"non-positive dimension"), ({"a10": 0}, b"non-positive dimension"),
                    ({"a11": 2}, b"square and odd"), ({"a12": 1}, b"square and odd"),
                    ({"a5": 34}, b"exceeds the row stride"), ({"a14": 16}, b"scratch smaller")]:
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, err)
    for args, msg in [((None, 2, 3, 8, 0, FAKE, None), b"bad argument"), ((FAKE, 2, 0, 8, 0, 2 * FAKE, None), b"bad argument"),
                      ((FAKE, 2, 3, 8, 1, FAKE, None), b"alias")]:
        rc = L.stp3_temporal_pair_mean(*args)
        assert rc == -1 and msg in L.stp3_last_error(), args
    # the scalar BatchNorm path widens the accepted domain but keeps refusing what cannot be right
    rc = L.stp3_bn_apply(FAKE, 100, 35, 34, FAKE, FAKE, FAKE, FAKE, None, 0, 1, 0.0, 0, 0, FAKE, 35, None, None, 0, None)
    assert rc == -1 and b"exceeds the row stride" in L.stp3_last_error()
    rc = L.stp3_bn_apply(FAKE, 100, 35, 35, FAKE, FAKE, FAKE, FAKE, None, 0, 1, 0.0, 0, 0, None, 0, FAKE, FAKE, 36, None)
    assert rc == -1 and b"bad bf16 planes" in L.stp3_last_error()
    rc = L.stp3_bn_bwd_apply(FAKE, 35, None, 0, FAKE, 35, FAKE, FAKE, FAKE, FAKE, FAKE, 100, 35, FAKE, 34, None, 0, None)
    assert rc == -1 and b"exceeds a row stride" in L.stp3_last_error()
