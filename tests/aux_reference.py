"""float64 reference of the EfficientNet trunk kernels and the memory-bound helpers of the dense path
(include/stp3_b200.h): stp3_effnet_stem, stp3_dw_fwd, stp3_se_gate (the gate and the packed per-image projection
weights), stp3_f32_to_hilo / stp3_hilo_to_f32 (bit-exact), stp3_spatial_sum, stp3_pool_bias, stp3_small_linear and
stp3_upsample2x_add.

Every function reads the raw buffers and arguments of one call (CPU or CUDA tensors) and evaluates the contract from the
stored inputs: hi + lo of the bf16 planes, the fp32 weights, biases and sums, the fp32 value of a float argument.  Next
to the values it returns `mag`, the sum of the magnitudes of the terms that make up each value: the scale a fixed-order
fp32 evaluation's round-off grows with."""
from typing import List, Optional, Tuple

import torch

F64 = torch.float64


def f32(v: float) -> float:
    """a Python float as the fp32 value a float argument of the C ABI receives"""
    return float(torch.tensor(v, dtype=torch.float32))


def planes(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    return hi.to(F64) + lo.to(F64)


# ------------------------------------------------------------------------------------------------ bf16 rounding
def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16, round to nearest, ties to even, by integer arithmetic on the fp32 bits (overflow gives inf, NaN
    stays a NaN)."""
    u = x.to(torch.float32).contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    r = torch.where(torch.isnan(x), (u >> 16) | 0x40, r) & 0xFFFF
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16).view(torch.bfloat16)


def split(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """the header's hi = bf16(x), lo = bf16(x - hi), the difference taken in fp32"""
    x = x.to(torch.float32)
    hi = bf16_rn(x)
    return hi, bf16_rn(x - hi.float())


def split_valid(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    """per element: hi is a bf16 nearest to hi + lo, i.e. |lo| <= half the gap from hi to its bf16 neighbour on lo's
    side -- what hi = bf16_rn(x), lo = bf16_rn(x - hi) guarantees.  (Ties count as valid: rounding lo can land hi + lo
    exactly halfway, e.g. x = 1 + 2^-8 + 2^-20.)  A hi rounded the wrong way moves hi + lo by less than the 2^-17 value
    allowance of the stored planes, so only this sees it.  Only finite hi are judged."""
    hb = hi.contiguous().view(torch.int16).to(torch.int32) & 0x7FFF          # |hi|
    as_f = lambda b: b.to(torch.int16).view(torch.bfloat16).to(F64)           # noqa: E731
    ahi = as_f(hb)
    up = as_f((hb + 1).clamp_max(0x7F80)) - ahi                               # gap away from zero
    down = torch.where(hb > 0, ahi - as_f((hb - 1).clamp_min(0)), up)         # gap toward zero
    lo64 = lo.to(F64)
    toward_zero = (lo64 != 0) & ((lo64 < 0) != (hi.to(F64) < 0)) & (hb > 0)
    return (lo64.abs() <= torch.where(toward_zero, down, up) / 2) | ~torch.isfinite(hi.float())


# ------------------------------------------------------------------------------------------------ windows
def _pad_nhwc(x: torch.Tensor, k: int, stride: int, pad_t: int, pad_l: int, Ho: int, Wo: int) -> torch.Tensor:
    """x (N, H, W, C) placed at (pad_t, pad_l) in zeros large enough for every tap of every output pixel"""
    N, H, W, C = x.shape
    Hp = max((Ho - 1) * stride + k, pad_t + H)
    Wp = max((Wo - 1) * stride + k, pad_l + W)
    xp = x.new_zeros((N, Hp, Wp, C))
    xp[:, pad_t:pad_t + H, pad_l:pad_l + W] = x
    return xp


def _tap(xp: torch.Tensor, ky: int, kx: int, stride: int, Ho: int, Wo: int) -> torch.Tensor:
    return xp[:, ky:ky + (Ho - 1) * stride + 1:stride, kx:kx + (Wo - 1) * stride + 1:stride]


def _swish(a: torch.Tensor) -> torch.Tensor:
    return a * torch.sigmoid(a)


# ------------------------------------------------------------------------------------------------ trunk
def stem(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, Ho: int, Wo: int, pad_t: int, pad_l: int,
         out_cstride: int) -> dict:
    """x (n, 3, H, W) fp32 NCHW, w (cout, 3, 3, 3) or (cout, 27), bias (cout) -> y (n, Ho, Wo, out_cstride): channels
    [0, cout) = swish(3x3 stride-2 convolution + bias), inputs outside the image zero; channels [cout, out_cstride) 0"""
    n = x.shape[0]
    cout = bias.numel()
    xp = _pad_nhwc(x.to(F64).permute(0, 2, 3, 1), 3, 2, pad_t, pad_l, Ho, Wo)
    w = w.to(F64).reshape(cout, 3, 3, 3)
    a = bias.to(F64).expand(n, Ho, Wo, cout).clone()
    mag = bias.to(F64).abs().expand(n, Ho, Wo, cout).clone()
    for ky in range(3):
        for kx in range(3):
            t = _tap(xp, ky, kx, 2, Ho, Wo)                     # (n, Ho, Wo, 3)
            a += t @ w[:, :, ky, kx].t()
            mag += t.abs() @ w[:, :, ky, kx].abs().t()
    y = a.new_zeros((n, Ho, Wo, out_cstride))
    y[..., :cout] = _swish(a)
    m = a.new_zeros((n, Ho, Wo, out_cstride))
    m[..., :cout] = mag
    return {"y": y, "mag": m}


def dw(x_hi: torch.Tensor, x_lo: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, k: int, stride: int, pad_t: int,
       pad_l: int, Ho: int, Wo: int, C: int) -> dict:
    """x planes (n, H, W, in_cstride), w (k*k, C), bias (C) -> y (n, Ho, Wo, C) = swish(depthwise conv + bias) of
    channels [0, C); sums (n, C) = the sum of y over the pixels.  sums_mag adds up, per pixel, the magnitude of the
    pre-activation's terms (what the error of each y scales with: swish can shrink y far below them) and |y| (what
    the summation's round-off scales with)"""
    x = planes(x_hi[..., :C], x_lo[..., :C])
    xp = _pad_nhwc(x, k, stride, pad_t, pad_l, Ho, Wo)
    w = w.to(F64).reshape(k * k, C)
    a = bias.to(F64).expand(x.shape[0], Ho, Wo, C).clone()
    mag = bias.to(F64).abs().expand(x.shape[0], Ho, Wo, C).clone()
    for ky in range(k):
        for kx in range(k):
            t = _tap(xp, ky, kx, stride, Ho, Wo)
            a += t * w[ky * k + kx]
            mag += (t * w[ky * k + kx]).abs()
    y = _swish(a)
    return {"y": y, "mag": mag, "sums": y.sum((1, 2)), "sums_mag": (mag + y.abs()).sum((1, 2))}


def se_layout(C: int, cout: int) -> Tuple[List[Tuple[int, int, int, int]], int]:
    """the chunks of stp3_se_gate's per-image block: [(first output channel, channels, bn, element offset)] and the
    block's size.  Chunks of 128 output channels, the last one 64 rows wide when it holds 64 or fewer, 128 otherwise;
    each [ceil(C / 64)][2 planes][bn][64]"""
    kb = -(-C // 64)
    chunks, off = [], 0
    for n0 in range(0, cout, 128):
        bn = 128 if cout - n0 > 64 else 64
        chunks.append((n0, min(128, cout - n0), bn, off))
        off += kb * 2 * bn * 64
    return chunks, off


def se_unpack(w_img: torch.Tensor, C: int, cout: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(n_img, elems) packed bf16 -> hi, lo (n_img, rows, ceil(C/64) * 64): row n = output channel n (the chunks stacked,
    their zero-padding rows included), column c = input channel c"""
    chunks, total = se_layout(C, cout)
    assert w_img.shape[1] >= total
    kb = -(-C // 64)
    his, los = [], []
    for n0, n, bn, off in chunks:
        blk = w_img[:, off:off + kb * 2 * bn * 64].reshape(-1, kb, 2, bn, 64)
        his.append(blk[:, :, 0].permute(0, 2, 1, 3).reshape(-1, bn, kb * 64))
        los.append(blk[:, :, 1].permute(0, 2, 1, 3).reshape(-1, bn, kb * 64))
    return torch.cat(his, 1), torch.cat(los, 1)


def se_gate(sums: torch.Tensor, C: int, inv_hw: float, w_r: torch.Tensor, b_r: torch.Tensor, w_e: torch.Tensor,
            b_e: torch.Tensor) -> dict:
    """sums (n_img, sums_stride): columns [0, C) read.  gate = sigmoid(w_e . swish(w_r . (sums * inv_hw) + b_r) + b_e);
    mag bounds the gate's sensitivity to an fp32 evaluation: 1/4 of the magnitudes of the logit's terms, the hidden
    values taken with the magnitudes of their own terms"""
    m = sums[:, :C].to(F64) * f32(inv_hw)
    h = m @ w_r.to(F64).t() + b_r.to(F64)
    h_mag = m.abs() @ w_r.to(F64).abs().t() + b_r.to(F64).abs()
    r = _swish(h)
    logit = r @ w_e.to(F64).t() + b_e.to(F64)
    mag = 0.25 * ((r.abs() + 1.1 * h_mag) @ w_e.to(F64).abs().t() + b_e.to(F64).abs())
    return {"gate": torch.sigmoid(logit), "mag": mag}


def se_weights(w_proj: torch.Tensor, gate: torch.Tensor, C: int, cout: int) -> torch.Tensor:
    """W_proj . diag(gate) of every image as (n_img, rows, ceil(C/64) * 64) in se_unpack's order, zero padded"""
    chunks, _ = se_layout(C, cout)
    rows = sum(bn for _, _, bn, _ in chunks)
    out = torch.zeros((gate.shape[0], rows, -(-C // 64) * 64), dtype=F64, device=gate.device)
    out[:, :cout, :C] = w_proj.to(F64).unsqueeze(0) * gate.to(F64).unsqueeze(1)
    return out


# ------------------------------------------------------------------------------------------------ layout glue
def f32_to_hilo(x: torch.Tensor, channels_last: int, n_img: int, C: int, H: int, W: int, cp: int):
    """x fp32 (n_img, C, H, W) or (n_img, H, W, C) -> hi, lo (n_img, H, W, cp), channels [C, cp) zero: bit-exact"""
    x = x.reshape(n_img, H, W, C) if channels_last else x.reshape(n_img, C, H, W).permute(0, 2, 3, 1)
    hi, lo = split(x)
    z = torch.zeros((n_img, H, W, cp - C), dtype=torch.bfloat16, device=x.device)
    return torch.cat([hi, z], -1), torch.cat([lo, z], -1)


def f32_to_plane(x: torch.Tensor, channels_last: int, n_img: int, C: int, H: int, W: int, cp: int,
                 mode: torch.dtype) -> torch.Tensor:
    """x fp32 (n_img, C, H, W) or (n_img, H, W, C) -> ONE plane (n_img, H, W, cp) of `mode` (torch.float16 /
    torch.bfloat16): torch's own rounding (to nearest even, overflow to +-inf, NaN kept), channels [C, cp) +0: bit-exact
    except for the NaN payloads"""
    x = x.reshape(n_img, H, W, C) if channels_last else x.reshape(n_img, C, H, W).permute(0, 2, 3, 1)
    z = torch.zeros((n_img, H, W, cp - C), dtype=mode, device=x.device)
    return torch.cat([x.to(mode), z], -1)


def hilo_to_f32(hi: torch.Tensor, lo: torch.Tensor, n_img: int, H: int, W: int, cstride: int, c_off: int, C: int):
    """planes (n_img, H, W, cstride), channels [c_off, c_off + C) -> (n_img, C, H, W) fp32 hi + lo, summed in fp32:
    bit-exact"""
    h = hi.reshape(n_img, H, W, cstride)[..., c_off:c_off + C].float()
    l = lo.reshape(n_img, H, W, cstride)[..., c_off:c_off + C].float()   # noqa: E741
    return (h + l).permute(0, 3, 1, 2).contiguous()


def spatial_sum(hi: torch.Tensor, lo: torch.Tensor, n_img: int, HW: int, cstride: int) -> dict:
    x = planes(hi, lo).reshape(n_img, HW, cstride)
    return {"sums": x.sum(1), "mag": x.abs().sum(1)}


# ------------------------------------------------------------------------------------------------ small dense layers
def _base(prior: Optional[torch.Tensor], bias: Optional[torch.Tensor], accumulate: bool, n: int, co: int, dev):
    """accumulate beats bias, bias beats 0"""
    if accumulate:
        return prior[:, :co].to(F64)
    if bias is not None:
        return bias[:co].to(F64).expand(n, co)
    return torch.zeros((n, co), dtype=F64, device=dev)


def pool_bias(sums: torch.Tensor, n_img: int, T: int, C: int, inv_hw: float, temporal: bool,
              const_vals: Optional[torch.Tensor], n_const: int, W1: torch.Tensor, b1: torch.Tensor, W2: torch.Tensor,
              bias: Optional[torch.Tensor], prior: Optional[torch.Tensor], accumulate: bool) -> dict:
    """sums (n_img, sums_stride) columns [0, C - n_const); const_vals (n_img, n_const); -> out (n_img, CO), the
    columns the call writes"""
    cs = C - n_const
    m = sums[:, :cs].to(F64) * f32(inv_hw)
    if n_const:
        m = torch.cat([m, const_vals.reshape(n_img, n_const).to(F64)], 1)
    if temporal:
        has_prev = (torch.arange(n_img, device=m.device) % T > 0).view(-1, 1)
        prev = torch.cat([m[:1], m[:-1]])
        m = torch.where(has_prev, (m + prev) / 2, m)
    W1, W2 = W1.to(F64).reshape(-1, C), W2.to(F64)
    CO = W2.shape[0]
    h = m @ W1.t() + b1.to(F64)
    v = h.clamp_min(0)
    base = _base(prior, bias, accumulate, n_img, CO, m.device)
    h_mag = m.abs() @ W1.abs().t() + b1.to(F64).abs()
    return {"out": base + v @ W2.t(), "mag": base.abs() + h_mag @ W2.abs().t()}


def small_linear(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], prior: Optional[torch.Tensor],
                 accumulate: bool) -> dict:
    """x (n, ci), W (co, ci) -> y (n, co) = base + W x"""
    x, W = x.to(F64), W.to(F64)
    base = _base(prior, bias, accumulate, x.shape[0], W.shape[0], x.device)
    return {"out": base + x @ W.t(), "mag": base.abs() + x.abs() @ W.abs().t()}


def _bilinear_src(n_out: int, n_in: int, dev):
    """source rows / columns and weights of align_corners=False x2: src = max((o + 0.5) / 2 - 0.5, 0), clamped"""
    src = ((torch.arange(n_out, dtype=F64, device=dev) + 0.5) * 0.5 - 0.5).clamp_min(0)
    i0 = src.floor().long()
    i1 = (i0 + 1).clamp_max(n_in - 1)
    f = src - i0
    return i0, i1, 1 - f, f


def upsample2x_add(x_hi, x_lo, n_img: int, h: int, w: int, C: int, s_hi=None, s_lo=None, s_coff: int = 0) -> dict:
    """x planes (n_img, h, w, x_cstride) channels [0, C) -> (n_img, 2h, 2w, C) bilinear x2 (+ skip channels
    [s_coff, s_coff + C) of (n_img, 2h, 2w, s_cstride))"""
    x = planes(x_hi[..., :C], x_lo[..., :C]).reshape(n_img, h, w, C)
    y0, y1, wy0, wy1 = _bilinear_src(2 * h, h, x.device)
    x0, x1, wx0, wx1 = _bilinear_src(2 * w, w, x.device)
    out = torch.zeros((n_img, 2 * h, 2 * w, C), dtype=F64, device=x.device)
    mag = torch.zeros_like(out)
    for yi, wy in ((y0, wy0), (y1, wy1)):
        for xi, wx in ((x0, wx0), (x1, wx1)):
            t = x[:, yi][:, :, xi] * (wy.view(-1, 1, 1) * wx.view(1, -1, 1))
            out += t
            mag += t.abs()
    if s_hi is not None:
        s = planes(s_hi[..., s_coff:s_coff + C], s_lo[..., s_coff:s_coff + C]).reshape(n_img, 2 * h, 2 * w, C)
        out += s
        mag += s.abs()
    return {"y": out, "mag": mag}
