"""Float64 reference of the stp3_conv_fwd contract (include/stp3_b200.h), evaluated from a PackedConv and the input's
bf16 hi/lo planes rather than from a PyTorch layer, so that it checks exactly what the kernel promises.  Runs on CPU or
CUDA tensors (per-tap float64 matmuls; on the device that is DGEMM, which uses no TF32).

  exact:  (x_hi + x_lo) . (w_hi + w_lo)                        the convolution of the values the planes carry
  model:  x_hi . w_hi + x_hi . w_lo + x_lo . w_hi               the three bf16 products the kernel issues
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


def tap_sum(x_hi: torch.Tensor, x_lo: torch.Tensor, pc: dense.PackedConv, *, cin_off: int = 0,
            frames: Optional[Tuple[int, int]] = None, out_hw: Optional[Tuple[int, int]] = None,
            model: bool = False) -> torch.Tensor:
    """Sum over pc.taps of the input window [cin_off, cin_off + cin_p) times the tap's weights, before bias and
    activation: (B*T, Ho, Wo, bn) float64.  Geometry as in dense.conv: frames (t0, T) of T_total, output size
    ceil(H / stride) unless out_hw is given."""
    B, Tt, H, W, _ = x_hi.shape
    t0, T = frames if frames is not None else (0, Tt)
    s = pc.stride
    Ho, Wo = out_hw if out_hw is not None else ((H + s - 1) // s, (W + s - 1) // s)
    xh = x_hi[..., cin_off:cin_off + pc.cin_p].double()
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
