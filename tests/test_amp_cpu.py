"""CPU: the one-plane (autocast) entry points refuse bad arguments before touching the device, the train path takes its
precision mode from the autocast state, and one-plane weights are packed as the kernels read them."""
import os

import torch

from stp3_b200 import _lib, dense
from stp3_b200 import dense_train as T

FAKE = 1 << 20   # a non-null, aligned device address: every call below is refused before it is dereferenced


def lib():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


def test_new_entry_points_refuse_bad_arguments():
    L = lib()
    BF, F16 = _lib.OPERAND_BF16, _lib.OPERAND_F16
    # stp3_conv_wgrad_plane
    ok = [F16, FAKE, 2, 14, 30, 64, 64, FAKE, 14, 30, 64, 64, 3, 3, 1, 1, 1, FAKE, 1 << 40, FAKE, None]

    def wg(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return L.stp3_conv_wgrad_plane(*a), L.stp3_last_error()
    for kw, msg in [({"a0": 0}, b"operand must be"), ({"a0": 3}, b"operand must be"), ({"a1": None}, b"null pointer"),
                    ({"a19": None}, b"null pointer"), ({"a2": 0}, b"non-positive dimension"),
                    ({"a14": 3}, b"stride must be 1 or 2"), ({"a16": 0}, b"dilation must be >= 1"),
                    ({"a5": 32}, b"exceeds the row stride"), ({"a18": 16}, b"scratch smaller")]:
        rc, err = wg(**kw)
        assert rc == -1 and msg in err, (kw, err)
    # stp3_conv3d_wgrad_plane
    ok3 = [BF, FAKE, 2, 3, 48, 64, 35, 35, FAKE, 35, 35, 2, 3, 3, FAKE, 1 << 40, FAKE, None]

    def wg3(**kw):
        a = list(ok3)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return L.stp3_conv3d_wgrad_plane(*a), L.stp3_last_error()
    for kw, msg in [({"a0": 0}, b"operand must be"), ({"a1": None}, b"null pointer"), ({"a3": 0}, b"non-positive"),
                    ({"a12": 2}, b"square and odd"), ({"a6": 34}, b"exceeds the row stride"),
                    ({"a15": 16}, b"scratch smaller")]:
        rc, err = wg3(**kw)
        assert rc == -1 and msg in err, (kw, err)
    # stp3_f32_to_plane
    for args, msg in [((None, 1, 2, 64, 8, 8, 64, F16, FAKE, None), b"bad argument"),
                      ((FAKE, 1, 2, 64, 8, 8, 32, F16, FAKE, None), b"bad argument"),
                      ((FAKE, 1, 2, 64, 8, 8, 64, 0, FAKE, None), b"operand must be"),
                      ((FAKE, 1, 70000, 64, 8, 8, 64, BF, FAKE, None), b"more than 65535")]:
        assert L.stp3_f32_to_plane(*args) == -1 and msg in L.stp3_last_error(), args
    # stp3_bn_apply_plane
    base = [FAKE, 100, 64, 64, FAKE, FAKE, FAKE, FAKE, None, 0, 1, 0.0, 0, 0, FAKE, 64, FAKE, 64, F16, None]

    def bn(**kw):
        a = list(base)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return L.stp3_bn_apply_plane(*a), L.stp3_last_error()
    for kw, msg in [({"a18": 0}, b"operand must be"), ({"a11": 1.0}, b"dropout p must be in [0, 1)"),
                    ({"a17": 36}, b"bad bf16 planes"), ({"a16": FAKE + 2}, b"bad bf16 planes"),
                    ({"a3": 32}, b"exceeds the row stride")]:
        rc, err = bn(**kw)
        assert rc == -1 and msg in err, (kw, err)
    # stp3_conv_fwd_plane: operand, outputs and the features it does not carry
    d = _lib.ConvDesc(B=1, T=1, H=8, W=8, in_cstride=64, cin=64, Ho=8, Wo=8, stride=1, ntaps=1, bn=64, n_valid=64,
                      f32_layout=1)

    def fwd(operand=F16, y=FAKE, **kw):
        for k, v in kw.items():
            setattr(d, k, v)
        rc = L.stp3_conv_fwd_plane(d, operand, FAKE, FAKE, FAKE, None, y, None)
        for k in kw:
            setattr(d, k, 0)
        return rc, L.stp3_last_error()
    for kw, msg in [(dict(operand=0), b"operand must be"), (dict(operand=3), b"operand must be"),
                    (dict(y=None), b"null pointer"), (dict(res_mode=1), b"no residual"), (dict(swish=1), b"no residual"),
                    (dict(w_img_stride=64 * 64 * 2), b"no residual"), (dict(bn=96), b"bn (padded output channels)")]:
        rc, err = fwd(**kw)
        assert rc == -1 and msg in err, (kw, err)


def test_mode_follows_the_autocast_state(monkeypatch):
    """amp_mode() reads the CUDA autocast state.  Without a GPU torch disables CUDA autocast regions, so the state is
    simulated here; tests/test_amp_train_gpu.py runs real ones."""
    assert T.amp_mode() is None
    state = {"enabled": True, "dtype": torch.float16}
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda dev="cuda": state["enabled"] and dev == "cuda")
    monkeypatch.setattr(torch, "get_autocast_dtype", lambda dev="cuda": state["dtype"])
    assert T.amp_mode() is torch.float16
    state["dtype"] = torch.bfloat16
    assert T.amp_mode() is torch.bfloat16
    state["dtype"] = torch.float32                          # not a 16-bit autocast: the fp32-equivalent path
    assert T.amp_mode() is None
    state.update(enabled=False, dtype=torch.float16)
    assert T.amp_mode() is None


def test_one_plane_packing():
    w = torch.randn(70, 35, 3, 3, dtype=torch.float64).float() * 1e-3
    w[0, 0, 1, 1] = 1e6                                       # beyond fp16: inf, as autocast's own cast of F.conv2d
    for plane in (torch.float16, torch.bfloat16):
        pc = dense.pack_conv(w, torch.zeros(70), plane=plane)
        assert pc.plane is plane and pc.w.dtype == plane and pc.w.shape == (9, 1, 128, 64)
        for i, (_, dy, dx) in enumerate(pc.taps):
            assert torch.equal(pc.w[i, 0, :70, :35].float(), w[:, :, dy + 1, dx + 1].to(plane).float())
            assert not pc.w[i, 0, 70:].any() and not pc.w[i, 0, :, 35:].any()
    assert torch.isinf(dense.pack_conv(w, torch.zeros(70), plane=torch.float16).w).any()
    hl = dense.pack_conv(w, torch.zeros(70))
    assert hl.plane is None and hl.w.shape == (9, 1, 2, 128, 64)
    pd = T.pack_dgrad(w, 1, 1, plane=torch.bfloat16)
    assert pd[0][1].plane is torch.bfloat16 and pd[0][1].w.shape == (9, 2, 64, 64)
