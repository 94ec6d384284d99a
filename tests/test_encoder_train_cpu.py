"""CPU: the train-mode encoder heads' oracle, the channel-window arithmetic of the upsample pair and the refusals that
need no device.

(a) The fp64 restatements (oracle/torch_encoder_train) against tests/golden/encoder_heads_train.npz, which the
    reference's own UpsamplingConcat and DeepLabHead produced in train mode (oracle/make_golden_encoder_train.py): outputs
    and running statistics to 1e-5, every gradient (parameters, r_lo, r_hi) to 1e-4 of the tensor's max, ReLU branches
    pinned where the fixture marks an input within round-off of zero.
(b) A numpy model of stp3_upsample2x_window_f32 / _bwd's thread -> (pixel, channel) map: with 1 or 4 channels per thread
    every element of the window is written once and nothing outside it; the model's forward equals F.interpolate and its
    adjoint the autograd gradient, for the encoder's windows and an unaligned one.
(c) The new C entry points and the modules refuse bad arguments before touching device memory."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import make_golden_encoder_train as MG
from oracle import torch_dense_train as TT
from oracle import torch_deeplab_train as TH
from oracle import torch_encoder_train as TE
from stp3_b200 import _lib
from stp3_b200.layers import convolutions as CV
from tests.test_abi import FAKE, lift_desc


# ------------------------------------------------------------------------------------------------ (a)
@pytest.mark.parametrize("name", ["uc", "feat", "depth"])
def test_fp64_train_oracle_matches_reference_fixture(name):
    golden = np.load("tests/golden/encoder_heads_train.npz")
    pre = name + "."
    head, up, mods = MG.make_modules(CV, name)
    mods.double()
    r_lo, r_hi = (t.double().requires_grad_(True) for t in MG.endpoints())
    calls = []

    def relu(t):
        k = len(calls)
        calls.append(k)
        m = (t.detach() > 0).reshape(-1)
        idx = torch.from_numpy(golden[f"{pre}relu{k}_idx"].astype(np.int64))
        m[idx] = torch.from_numpy(golden[f"{pre}relu{k}_pos"])
        return t * m.view(t.shape).to(t.dtype)
    if head is None:
        out = TE.upsampling_concat_train(r_hi, r_lo, up, relu=relu)
    else:
        mask = TH.dropout_keep_mask((MG.M, MG.HIDDEN, MG.H, MG.W), int(golden["mask_seed"]), float(golden["p"]))
        out = TE.encoder_head_train(r_lo, r_hi, head, up, relu=relu, dropout_mask=mask)
    assert len(calls) == int(golden[pre + "n_relu"])
    G = TT.upstream_grads({"out": out}, seed=MG.GRAD_SEED)["out"]
    (out * G.double()).sum().backward()
    flat = out.detach().reshape(-1)
    s = golden[pre + "out_s"]
    e = np.abs(flat[TT.sample_index(pre + "out", flat.numel(), len(s))].numpy() - s).max() / golden[pre + "out_amax"]
    assert e < 1e-5, e
    for k, b in mods.named_buffers():
        want = golden[pre + k]
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(want), k
            continue
        e = np.abs(b.numpy() - want).max() / np.abs(want).max()
        assert e < 1e-5, (k, e)
    for k, p in list(mods.named_parameters()) + [("r_lo", r_lo), ("r_hi", r_hi)]:
        flat = p.grad.reshape(-1)
        s = golden[f"{pre}grad_{k}_s"]
        idx = TT.sample_index(f"{pre}grad.{k}", flat.numel(), len(s))
        e = np.abs(flat[idx].numpy() - s).max() / golden[f"{pre}grad_{k}_amax"]
        assert e < 1e-4, (k, e)


# ------------------------------------------------------------------------------------------------ (b)
def up_coord(o, n):
    f = max((o + 0.5) * 0.5 - 0.5, 0.0)
    i0 = int(f)
    return i0, min(i0 + 1, n - 1), 1.0 - (f - i0), f - i0


def vec_width(C, cstride, coff):
    """The kernels' rule (for 16-byte aligned base pointers): 4 channels per thread or 1."""
    return 4 if C % 4 == 0 and cstride % 4 == 0 and coff % 4 == 0 else 1


def window_fwd_model(x, y, coff):
    """x (N,h,w,C) float64 -> writes y (N,2h,2w,Cy)[..., coff:coff+C] thread by thread; returns the write counts."""
    N, h, w, C = x.shape
    cs = y.shape[-1]
    V = vec_width(C, cs, coff)
    yf, count = y.reshape(-1), np.zeros(y.size, dtype=np.int64)
    for i in range(N * 2 * h * 2 * w * (C // V)):
        c = (i % (C // V)) * V
        orow = i // (C // V)
        ox, oy, img = orow % (2 * w), orow // (2 * w) % (2 * h), orow // (2 * w) // (2 * h)
        y0, y1, wy0, wy1 = up_coord(oy, h)
        x0, x1, wx0, wx1 = up_coord(ox, w)
        for k in range(V):
            b = x[img, :, :, c + k]
            dst = orow * cs + coff + c + k
            yf[dst] = wy0 * (wx0 * b[y0, x0] + wx1 * b[y0, x1]) + wy1 * (wx0 * b[y1, x0] + wx1 * b[y1, x1])
            count[dst] += 1
    return count.reshape(y.shape)


def window_bwd_model(gy, coff, C):
    """gy (N,2h,2w,Cy) float64 -> dense gx (N,h,w,C): the gather over outputs 2i-1 .. 2i+2, thread by thread."""
    N, H2, W2, cs = gy.shape
    h, w = H2 // 2, W2 // 2
    V = vec_width(C, cs, coff)
    gx, count = np.zeros(N * h * w * C), np.zeros(N * h * w * C, dtype=np.int64)
    gf = gy.reshape(-1)

    def weight(o, n, i):
        i0, i1, w0, w1 = up_coord(o, n)
        return (w0 if i0 == i else 0.0) + (w1 if i1 == i else 0.0)
    for i in range(N * h * w * (C // V)):
        c = (i % (C // V)) * V
        r = i // (C // V)
        ix, iy, img = r % w, r // w % h, r // w // h
        for k in range(V):
            acc = 0.0
            for oy in range(max(2 * iy - 1, 0), min(2 * iy + 2, 2 * h - 1) + 1):
                row = 0.0
                for ox in range(max(2 * ix - 1, 0), min(2 * ix + 2, 2 * w - 1) + 1):
                    row += weight(ox, w, ix) * gf[((img * 2 * h + oy) * 2 * w + ox) * cs + coff + c + k]
                acc += weight(oy, h, iy) * row
            gx[i * V + k] = acc
            count[i * V + k] += 1
    assert (count == 1).all()
    return gx.reshape(N, h, w, C)


@pytest.mark.parametrize("cf,cc", [(56, 160), (40, 112), (3, 5)])
def test_channel_window_arithmetic(cf, cc):
    N, h, w = 2, 3, 2
    assert vec_width(cc, cf + cc, cf) == (1 if (cf, cc) == (3, 5) else 4)
    rng = np.random.default_rng(cf)
    x = rng.standard_normal((N, h, w, cc))
    y = np.full((N, 2 * h, 2 * w, cf + cc), np.nan)
    count = window_fwd_model(x, y, cf)
    assert (count[..., cf:] == 1).all() and (count[..., :cf] == 0).all() and np.isnan(y[..., :cf]).all()
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.interpolate(xt, scale_factor=2, mode="bilinear", align_corners=False)
    assert np.abs(y[..., cf:] - ref.detach().permute(0, 2, 3, 1).numpy()).max() < 1e-12
    gy = rng.standard_normal(y.shape)
    ref.backward(torch.from_numpy(gy[..., cf:]).permute(0, 3, 1, 2))
    gx = window_bwd_model(gy, cf, cc)
    assert np.abs(gx - xt.grad.permute(0, 2, 3, 1).numpy()).max() < 1e-12


# ------------------------------------------------------------------------------------------------ (c)
def test_new_entry_points_refuse_bad_arguments():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    cl = lift_desc(feat_layout=1)
    big = 1 << 40
    assert L.stp3_lift_splat_bwd_cl(lift_desc(), FAKE, FAKE, FAKE, FAKE, big, FAKE, FAKE, None) == -1
    assert b"feat must be channels-last" in L.stp3_last_error()
    for args in ((None, FAKE, FAKE, FAKE, big, FAKE), (FAKE, None, FAKE, FAKE, big, FAKE),
                 (FAKE, FAKE, FAKE, None, big, FAKE), (FAKE, FAKE, FAKE, FAKE, big, None)):
        assert L.stp3_lift_splat_bwd_cl(cl, *args, FAKE, None) == -1, args
        assert b"null pointer" in L.stp3_last_error()
    assert L.stp3_lift_splat_bwd_cl(cl, FAKE, FAKE, FAKE, FAKE, 16, FAKE, FAKE, None) != 0
    assert b"scratch too small" in L.stp3_last_error()
    assert L.stp3_lift_splat_bwd_cl(lift_desc(feat_layout=1, C=63), FAKE, FAKE, FAKE, FAKE, big, FAKE, FAKE, None) == -1
    assert b"C must be even" in L.stp3_last_error()
    assert L.stp3_lift_splat_bwd_cl(lift_desc(feat_layout=1, S=9), FAKE, FAKE, FAKE, FAKE, big, FAKE, FAKE, None) == -1
    assert b"receptive field S=9" in L.stp3_last_error()
    # the window must lie inside the row
    assert L.stp3_upsample2x_window_f32(FAKE, 2, 14, 30, 160, FAKE, 216, 60, None) == -1
    assert b"outside rows of 216" in L.stp3_last_error()
    assert L.stp3_upsample2x_window_bwd(FAKE, 216, -4, 2, 14, 30, 160, FAKE, None) == -1
    assert b"outside rows of 216" in L.stp3_last_error()
    assert L.stp3_upsample2x_window_f32(None, 2, 14, 30, 160, FAKE, 216, 56, None) == -1
    assert L.stp3_upsample2x_window_bwd(FAKE, 216, 56, 2, 0, 30, 160, FAKE, None) == -1


def test_modules_refuse_without_a_device():
    from stp3_b200.config import get_cfg
    from stp3_b200.models.encoder import Encoder
    up = CV.UpsamplingConcat(216, 64).train()
    x_up, x = torch.zeros(2, 160, 4, 6), torch.zeros(2, 56, 8, 12)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        up(x_up, x)
    with pytest.raises(ValueError, match="channels_last is the train path's"):
        up.eval()(x_up, x, channels_last=True)
    with pytest.raises(NotImplementedError, match="SyncBatchNorm"):
        torch.nn.SyncBatchNorm.convert_sync_batchnorm(CV.UpsamplingConcat(216, 64)).train()(x_up, x)
    for attr, match in (("momentum", "momentum=None"), ("track_running_stats", "track_running_stats=False")):
        bad = CV.UpsamplingConcat(216, 64).train()
        setattr(bad.conv[4], attr, None if attr == "momentum" else False)
        with pytest.raises(NotImplementedError, match=match):
            bad(x_up, x)
    enc = Encoder(get_cfg().MODEL.ENCODER, D=48, backbone=torch.nn.Identity()).eval()
    assert enc.heads_training() is False
    assert enc.train_heads() is enc and enc.heads_training() is True and not enc.backbone.training
    enc.depth_layer_2.eval()
    with pytest.raises(RuntimeError, match="mixed train / eval"):
        enc.heads_training()
    assert enc.train_heads(False).heads_training() is False
