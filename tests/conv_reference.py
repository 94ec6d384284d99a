"""Float64 reference of the stp3_conv_fwd contract (include/stp3_b200.h), evaluated from a PackedConv and the input's
bf16 hi/lo planes rather than from a PyTorch layer, so that it checks exactly what the kernel promises.  Runs on CPU or
CUDA tensors (per-tap float64 matmuls; on the device that is DGEMM, which uses no TF32).

  exact:  (x_hi + x_lo) . (w_hi + w_lo)                        the convolution of the values the planes carry
  model:  x_hi . w_hi + x_hi . w_lo + x_lo . w_hi               the three bf16 products the kernel issues

One-plane operands (stp3_conv_fwd_plane: x and w each ONE fp16 / bf16 plane, pc.plane set, x_lo None) carry their
values exactly and the kernel issues one product per term, so the exact convolution of the plane values is also the
model: one fp64 tap sum serves both.  `absolute` sums |x| . |w| instead, the magnitude an fp32 accumulation's rounding
is measured against.
"""
from typing import Optional, Tuple

import torch

from stp3_b200 import dense


def unpack_weights(pc: dense.PackedConv) -> Tuple[torch.Tensor, torch.Tensor]:
    """pc.w [ntaps][cin_p/64][2][bn][64] bf16 -> (w_hi, w_lo) float64 (ntaps, bn, cin_p)."""
    nt, kbs, _, bn, kb = pc.w.shape
    hi = pc.w[:, :, 0].permute(0, 2, 1, 3).reshape(nt, bn, kbs * kb).double()
    lo = pc.w[:, :, 1].permute(0, 2, 1, 3).reshape(nt, bn, kbs * kb).double()
    return hi, lo


def unpack_plane(pc: dense.PackedConv) -> torch.Tensor:
    """one-plane pc.w [ntaps][cin_p/64][bn][64] fp16 / bf16 -> float64 (ntaps, bn, cin_p)"""
    nt, kbs, bn, kb = pc.w.shape
    return pc.w.permute(0, 2, 1, 3).reshape(nt, bn, kbs * kb).double()


def shifted(x: torch.Tensor, dt: int, dy: int, dx: int, t0: int, T: int, Ho: int, Wo: int, s: int) -> torch.Tensor:
    """x (B, T_total, H, W, C) -> (B, T, Ho, Wo, C): x[b, t0 + t + dt, oy*s + dy, ox*s + dx], zero outside the tensor."""
    B, Tt, H, W, C = x.shape
    out = x.new_zeros((B, T, Ho, Wo, C))
    t_lo, t_hi = max(0, -t0 - dt), min(T, Tt - t0 - dt)
    y_lo, y_hi = max(0, (-dy + s - 1) // s), min(Ho, (H - 1 - dy) // s + 1)
    x_lo, x_hi = max(0, (-dx + s - 1) // s), min(Wo, (W - 1 - dx) // s + 1)
    if t_lo < t_hi and y_lo < y_hi and x_lo < x_hi:
        out[:, t_lo:t_hi, y_lo:y_hi, x_lo:x_hi] = x[:, t0 + t_lo + dt:t0 + t_hi + dt,
                                                    y_lo * s + dy:(y_hi - 1) * s + dy + 1:s,
                                                    x_lo * s + dx:(x_hi - 1) * s + dx + 1:s]
    return out


def tap_sum(x_hi: torch.Tensor, x_lo: Optional[torch.Tensor], pc: dense.PackedConv, *, cin_off: int = 0,
            frames: Optional[Tuple[int, int]] = None, out_hw: Optional[Tuple[int, int]] = None,
            model: bool = False, absolute: bool = False) -> torch.Tensor:
    """Sum over pc.taps of the input window [cin_off, cin_off + cin_p) times the tap's weights, before bias and
    activation: (B*T, Ho, Wo, bn) float64.  Geometry as in dense.conv: frames (t0, T) of T_total, output size
    ceil(H / stride) unless out_hw is given.  One-plane pc (pc.plane set): x_hi is the plane and x_lo None; `model`
    changes nothing and `absolute` sums the magnitudes of the terms."""
    B, Tt, H, W, _ = x_hi.shape
    t0, T = frames if frames is not None else (0, Tt)
    s = pc.stride
    Ho, Wo = out_hw if out_hw is not None else ((H + s - 1) // s, (W + s - 1) // s)
    xh = x_hi[..., cin_off:cin_off + pc.cin_p].double()
    if pc.plane is not None:
        assert x_lo is None and x_hi.dtype == pc.plane, (x_hi.dtype, pc.plane)
        w = unpack_plane(pc).to(xh.device)
        if absolute:
            xh, w = xh.abs(), w.abs()
        acc = xh.new_zeros((B, T, Ho, Wo, pc.bn))
        for i, (dt, dy, dx) in enumerate(pc.taps):
            acc += shifted(xh, dt, dy, dx, t0, T, Ho, Wo, s) @ w[i].t()
        return acc.reshape(B * T, Ho, Wo, pc.bn)
    assert not absolute, "absolute: one-plane operands only"
    xl = x_lo[..., cin_off:cin_off + pc.cin_p].double()
    wh, wl = unpack_weights(pc)
    wh, wl = wh.to(xh.device), wl.to(xh.device)
    acc = xh.new_zeros((B, T, Ho, Wo, pc.bn))
    for i, (dt, dy, dx) in enumerate(pc.taps):
        ah = shifted(xh, dt, dy, dx, t0, T, Ho, Wo, s)
        al = shifted(xl, dt, dy, dx, t0, T, Ho, Wo, s)
        if model:
            acc += ah @ wh[i].t() + ah @ wl[i].t() + al @ wh[i].t()
        else:
            acc += (ah + al) @ (wh[i] + wl[i]).t()
    return acc.reshape(B * T, Ho, Wo, pc.bn)


def join(h: dense.HL) -> torch.Tensor:
    return h.hi.double() + h.lo.double()


def epilogue(acc: torch.Tensor, pc: dense.PackedConv, kw: dict) -> dict:
    """Outputs stp3_conv_fwd writes for the accumulator `acc` (B*T, Ho, Wo, bn) and the keyword arguments of dense.conv
    (tensors as given to the call).  Returns {name: float64 tensor}: 'y' / 'y2' the stored hi/lo channel windows,
    'f32' the fp32 output in its layout, 'head<k>' the fused head planes (B*T, Ho, Wo), 'col_sums' (B*T, 64)."""
    n_img, Ho, Wo, bn = acc.shape
    dev = acc.device
    ib = kw.get("img_bias")
    v = acc + (ib.double().to(dev).view(n_img, 1, 1, bn) if ib is not None else pc.bias.double().to(dev))
    res = kw.get("residual")
    relu = torch.zeros(bn, dtype=torch.bool, device=dev)
    relu[:] = bool(kw.get("relu", False))
    if kw.get("out2") is not None:
        relu[64:] = bool(kw.get("relu2", False))
    act = lambda t: torch.where(relu, t.clamp_min(0.0), t)      # noqa: E731
    if res is not None:
        r = join(res).to(dev).reshape(n_img, Ho, Wo, -1)
        rc = kw.get("res_coff", 0)
        r = r[..., rc:rc + bn]
        v = act(v) + r if kw.get("res_after_act", False) else act(v + r)
    else:
        v = act(v)
    out = {}
    if kw.get("out") is not None:
        n_store = kw.get("n_store", 0) or bn
        out["y"] = v[..., :n_store]
    if kw.get("out2") is not None:
        out["y2"] = v[..., 64:64 + (kw.get("n_store2", 0) or 64)]
    if kw.get("out_f32") is not None:
        nv = kw["n_valid"]
        f = v[..., :nv]
        if kw.get("out_f32_nhwc", False):
            out["f32"] = f
        else:
            out["f32"] = (torch.sigmoid(f) if kw.get("sigmoid", False) else f).permute(0, 3, 1, 2)
    head = kw.get("head")
    if head is not None:
        h = v @ head["w"].double().to(dev).t() + head["b"].double().to(dev)
        for k in range(h.shape[-1]):
            hk = h[..., k]
            out[f"head{k}"] = torch.sigmoid(hk) if (int(head.get("sigmoid_mask", 0)) >> k) & 1 else hk
    if kw.get("col_sums") is not None:
        out["col_sums"] = v.sum(dim=(1, 2))
    return out


def tiling(pc: dense.PackedConv, geom: Tuple[int, ...], cfg: Tuple[int, int], *, in_cstride: int, cin_off: int = 0,
           t0: int = 0, n_store: int = 0, one_block: bool = False, w_img_stride: int = 0, operand: int = 0,
           n_sm: int = 132) -> dict:
    """How the library runs a dense.conv call with tiling cfg = (n_sub, group): stp3_conv_tiling_op on the descriptor
    dense.conv builds (geom = (B, T_total, T, H, W, Ho, Wo); one_block: a fused head or a second destination, which
    drop the 64-column blocks; w_img_stride: per-image weights, which always stream).  -> the stp3_conv_tiling_info fields and `fullk` (the K range covers every 16-channel
    step of the first and last K blocks: conv_igemm_kernel's FULLK)."""
    import ctypes

    from stp3_b200 import _lib
    B, Tt, T, H, W, Ho, Wo = geom
    d = _lib.ConvDesc()
    d.B, d.T, d.H, d.W, d.T_total, d.t0 = B, T, H, W, Tt, t0
    d.in_cstride, d.cin_off, d.cin = in_cstride, cin_off, pc.cin_p
    d.Ho, d.Wo, d.stride, d.ntaps = Ho, Wo, pc.stride, len(pc.taps)
    for i, (dt, dy, dx) in enumerate(pc.taps):
        d.taps[i][0], d.taps[i][1], d.taps[i][2] = dt, dy, dx
    d.bn, d.n_cols, d.k_lo, d.k_hi, d.n_store = pc.bn, pc.cout, pc.k_lo, pc.k_hi, n_store
    d.w_img_stride = w_img_stride
    group = cfg[1]
    d.tune_n_sub, d.tune_group = cfg[0], group & ~dense.BLOCKS64
    d.tune_bn = 64 if group & dense.BLOCKS64 and not one_block else 0
    info = _lib.ConvTilingInfo()
    code = _lib.lib().stp3_conv_tiling_op(ctypes.byref(d), n_sm, operand, ctypes.byref(info))
    _lib.check(code, "stp3_conv_tiling_op")
    out = {k: getattr(info, k) for k, _ in _lib.ConvTilingInfo._fields_}
    kb = pc.cin_p // dense.KB
    k_lo, k_hi = (pc.k_lo, pc.k_hi) if pc.k_hi > 0 else (0, pc.cin_p)
    out["fullk"] = k_lo // 16 == 0 and (k_hi - (kb - 1) * dense.KB) // 16 == 4
    return out
