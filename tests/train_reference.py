"""float64 reference of the train-mode entry points of stp3_b200/csrc/train_kernels.cu (include/stp3_b200.h "Train mode").

Every function reads exactly what the kernel reads (the fp32 operands, and for the elementwise kernels the kernel's own
fp32 statistics) and evaluates the header's formula in float64, on the CPU or on CUDA (fp64 matmuls: DGEMM, no TF32).
Tensors are dense channels-last; the callers cut channel windows out of wider rows.

Besides the exact value, most functions return the magnitude the kernel's fp32 rounding is measured against: the sum of
the absolute values of the terms (an elementwise bar of a few ulps of that is what a correct fp32 evaluation meets), and
for the weight gradient the "model" value: the three bf16 products g_hi x_hi + g_hi x_lo + g_lo x_hi the tensor cores
issue, with the planes split like ptx::split_hilo (round to nearest, then the remainder to nearest).  The one-plane
(autocast) kernels read fp16 / bf16 values exactly and issue one product each, so their fp64 product of the rounded
values is both the exact result and the model (wgrad with `plane`)."""
from typing import List, Optional, Sequence

import numpy as np
import torch

from stp3_b200 import dense


def _d(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float64)


# ------------------------------------------------------------------------------------------------ weight gradient
def wgrad_split(P: int, ntaps: int, cout: int, cin: int):
    """(splits, pixels per split) of the weight gradient's K split (train_kernels.cu wgrad_splits / launch_wgrad):
    about 4 CTAs per SM of an H100 over the 64 x 64 output tiles, at least 256 pixels per split, per rounded up to 64.
    Splits past ceil(P / per) are empty and store zeros."""
    tiles = ntaps * -(-cout // 64) * -(-cin // 64)
    n = min(max(min((132 * 4 + tiles - 1) // tiles, (P + 255) // 256), 1), 1024)
    per = -(-P // n)
    return n, -(-per // 64) * 64


def _shift(x: torch.Tensor, dy: int, dx: int, dt: int, stride: int, Ho: int, Wo: int, T: int) -> torch.Tensor:
    """x (n_img, H, W, C) read at (img + dt, oy * stride + dy, ox * stride + dx) for every output pixel, zeros outside
    the image and outside the sample (img % T + dt < 0) -> (n_img, Ho, Wo, C)"""
    n, H, W, C = x.shape
    dev = x.device
    iy = torch.arange(Ho, device=dev) * stride + dy
    ix = torch.arange(Wo, device=dev) * stride + dx
    img = torch.arange(n, device=dev)
    vy, vx, vi = (iy >= 0) & (iy < H), (ix >= 0) & (ix < W), (img % T) + dt >= 0
    out = x[(img + dt).clamp(0, n - 1)][:, iy.clamp(0, H - 1)][:, :, ix.clamp(0, W - 1)]
    mask = vi.view(-1, 1, 1) & vy.view(1, -1, 1) & vx.view(1, 1, -1)
    return out * mask.unsqueeze(-1).to(out.dtype)


def wgrad(x: torch.Tensor, g: torch.Tensor, kh: int, kw: int, stride: int = 1, pad: int = 0, dil: int = 1,
          kt: int = 1, T: int = 1, model: bool = False, plane: Optional[torch.dtype] = None) -> torch.Tensor:
    """dw (cout, cin, kt, kh, kw) of stp3_conv_wgrad (kt = T = 1) or stp3_conv3d_wgrad (n_img = B * T frames,
    frame-major within a sample; time tap it reads frame t + it - (kt - 1)): x (n_img, H, W, cin) and g (n_img, Ho, Wo,
    cout) fp32.  model: the three bf16 products of the kernel instead of the exact product of the fp32 values.
    plane (torch.float16 / torch.bfloat16): stp3_conv_wgrad_plane / stp3_conv3d_wgrad_plane, the product of x and g
    rounded to that type (torch's rounding, as stp3_f32_to_plane; a plane passed in stays as it is)."""
    n, Ho, Wo, cout = g.shape
    cin = x.shape[-1]
    if plane is not None:
        pairs = [(g.to(plane), x.to(plane))]
    elif model:
        (xh, xl), (gh, gl) = dense.split_hilo(x.float()), dense.split_hilo(g.float())
        pairs = [(gh, xh), (gh, xl), (gl, xh)]
    else:
        pairs = [(g, x)]
    pairs = [(_d(a).reshape(-1, cout), _d(b)) for a, b in pairs]
    dw = torch.zeros((cout, cin, kt, kh, kw), dtype=torch.float64, device=x.device)
    for it in range(kt):
        for ky in range(kh):
            for kx in range(kw):
                for a, b in pairs:
                    xs = _shift(b, ky * dil - pad, kx * dil - pad, it - (kt - 1), stride, Ho, Wo, T)
                    dw[:, :, it, ky, kx] += a.t() @ xs.reshape(-1, cin)
    return dw


# ------------------------------------------------------------------------------------------------ BatchNorm
def bn_stats(x: torch.Tensor, eps: float, momentum: float, run_mean: Optional[torch.Tensor] = None,
             run_var: Optional[torch.Tensor] = None) -> dict:
    """stp3_bn_stats of x (n_pix, C) fp32: batch mean, biased variance, invstd = 1 / sqrt(var + eps), and the running
    statistics (1 - momentum) r + momentum b with the unbiased variance var * n / (n - 1) (n = 1: var)."""
    xd = _d(x)
    n = xd.shape[0]
    mean = xd.mean(0)
    var = ((xd - mean) ** 2).mean(0)
    out = {"mean": mean, "var": var, "invstd": 1.0 / torch.sqrt(var + float(np.float32(eps))),
           "abs_mean": xd.abs().mean(0), "sq_mean": (xd ** 2).mean(0)}
    if run_mean is not None:
        m = float(np.float32(momentum))
        unb = var * n / (n - 1) if n > 1 else var
        out["run_mean"] = (1 - m) * _d(run_mean) + m * mean
        out["run_var"] = (1 - m) * _d(run_var) + m * unb
    return out


def _philox_round(c0, c1, c2, c3, k0, k1):
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    p0, p1 = c0.astype(np.uint64) * m0, c2.astype(np.uint64) * m1
    hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0


def philox4x32_10(key: Sequence[int], ctr: np.ndarray) -> np.ndarray:
    """Philox-4x32-10 (Salmon et al., SC'11) of counters ctr (..., 4) uint32 under key (k0, k1) -> (..., 4) uint32:
    ten rounds of the two multiplications by 0xD2511F53 / 0xCD9E8D57, the key bumped by (0x9E3779B9, 0xBB67AE85)
    between rounds."""
    ctr = np.asarray(ctr, dtype=np.uint32)
    c = [ctr[..., i].copy() for i in range(4)]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for _ in range(10):
            c = list(_philox_round(*c, k0, k1))
            k0, k1 = np.uint32(k0 + np.uint32(0x9E3779B9)), np.uint32(k1 + np.uint32(0xBB67AE85))
    return np.stack(c, axis=-1)


def dropout_keep(seed: int, offset: int, n_pix: int, C: int, p: float) -> np.ndarray:
    """Keep bits (n_pix, C) of stp3_bn_apply: element e = offset + pixel * C + c keeps when word e % 4 of
    Philox-4x32-10(key = seed, counter = (e / 4, 0)) (64-bit values as (low, high) 32-bit words), read as
    (word >> 8) / 2^24, is >= p."""
    e = np.uint64(offset) + np.arange(n_pix * C, dtype=np.uint64)
    q = e >> np.uint64(2)
    ctr = np.stack([(q & np.uint64(0xFFFFFFFF)).astype(np.uint32), (q >> np.uint64(32)).astype(np.uint32),
                    np.zeros_like(q, dtype=np.uint32), np.zeros_like(q, dtype=np.uint32)], axis=-1)
    r = philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), ctr)
    w = np.take_along_axis(r, (e & np.uint64(3)).astype(np.int64)[:, None], axis=1)[:, 0]
    u = (w >> np.uint32(8)).astype(np.float64) / 2.0 ** 24
    return (u >= float(np.float32(p))).reshape(n_pix, C)


def dropout_scale(p: float) -> float:
    """the kernel's fp32 1 / (1 - p)"""
    one = np.float32(1.0)
    return float(one / (one - np.float32(p)))


def bn_apply(x, mean, invstd, gamma, beta, res=None, relu=False, p=0.0, seed=0, offset=0) -> dict:
    """stp3_bn_apply of x (n_pix, C) with the kernel's fp32 mean / invstd -> y (fp64), the keep bits (None without
    dropout) and the magnitude |xhat gamma| + |beta| + |res| of the terms (times the dropout scale)."""
    t = (_d(x) - _d(mean)) * _d(invstd) * _d(gamma) + _d(beta)
    mag = ((_d(x) - _d(mean)) * _d(invstd) * _d(gamma)).abs() + _d(beta).abs()
    if res is not None:
        t, mag = t + _d(res), mag + _d(res).abs()
    y = t.clamp_min(0.0) if relu else t
    keep = None
    if p > 0:
        n, C = x.shape
        keep = torch.from_numpy(dropout_keep(seed, offset, n, C, p)).to(x.device)
        s = dropout_scale(p)
        y, mag = torch.where(keep, y * s, torch.zeros_like(y)), mag * s
    return {"y": y, "keep": keep, "mag": mag}


def bn_apply_plane(y: torch.Tensor, cs: int, mode: torch.dtype) -> torch.Tensor:
    """the plane of stp3_bn_apply_plane: y (n_pix, C) fp32 as stp3_bn_apply stores it, rounded by torch's .to(mode),
    in rows of cs channels whose channels [C, cs) are +0"""
    n, C = y.shape
    out = torch.zeros((n, cs), dtype=mode, device=y.device)
    out[:, :C] = y.to(mode)
    return out


def _masked(g, y):
    gd = _d(g)
    return gd if y is None else torch.where(y > 0, gd, torch.zeros_like(gd))


def bn_bwd_reduce(g, y, x, mean, invstd) -> dict:
    """stp3_bn_bwd_reduce: sum_g = sum g', sum_gxhat = sum g' xhat (x given), g' = g where y > 0 (y given), xhat from
    the kernel's fp32 mean / invstd; with the sums of the term magnitudes."""
    gm = _masked(g, y)
    out = {"sum_g": gm.sum(0), "mag_g": gm.abs().sum(0)}
    if x is not None:
        xh = (_d(x) - _d(mean)) * _d(invstd)
        out["sum_gx"], out["mag_gx"] = (gm * xh).sum(0), (gm * xh).abs().sum(0)
    return out


def bn_bwd_apply(g, y, x, mean, invstd, gamma, sum_g, sum_gx) -> dict:
    """stp3_bn_bwd_apply: dx = gamma invstd (g' - sum_g / n - xhat sum_gxhat / n) from the kernel's fp32 statistics and
    sums, g' and the term magnitude."""
    n = x.shape[0]
    gm = _masked(g, y)
    xh = (_d(x) - _d(mean)) * _d(invstd)
    a = _d(gamma) * _d(invstd)
    dx = a * (gm - _d(sum_g) / n - xh * _d(sum_gx) / n)
    mag = a.abs() * (gm.abs() + _d(sum_g).abs() / n + (xh * _d(sum_gx)).abs() / n)
    return {"dx": dx, "g_masked": gm, "mag": mag}


def image_channel_sums(x: torch.Tensor) -> dict:
    """stp3_image_channel_sums of x (n_img, hw, C) -> sums (n_img, C) and the sums of magnitudes"""
    return {"sums": _d(x).sum(1), "mag": _d(x).abs().sum(1)}


# ------------------------------------------------------------------------------------------------ small kernels
def temporal_pair_mean(m: torch.Tensor, adjoint: bool = False) -> dict:
    """stp3_temporal_pair_mean: m (B, T, C) -> (B, T + 1, C); adjoint: m (B, T + 1, C) -> (B, T, C)"""
    md = _d(m)
    if not adjoint:                           # the end frames as (m[0] + m[0]) / 2 and (m[T-1] + m[T-1]) / 2: exact
        a = torch.cat([md[:, :1], md[:, :-1], md[:, -1:]], 1)
        b = torch.cat([md[:, :1], md[:, 1:], md[:, -1:]], 1)
        return {"out": 0.5 * (a + b), "mag": 0.5 * (a.abs() + b.abs())}
    T = md.shape[1] - 1
    c = torch.full((T,), 0.5, dtype=torch.float64, device=m.device)
    c[0] = 1.0
    nxt = torch.cat([0.5 * md[:, 1:T], md[:, T:T + 1]], 1)
    out = c.view(1, -1, 1) * md[:, :T] + nxt
    return {"out": out, "mag": (c.view(1, -1, 1) * md[:, :T]).abs() + nxt.abs()}


def upsample_matrix(n: int, device=None) -> torch.Tensor:
    """(2n, n) weights of bilinear x2 with align_corners=False along one axis: source (o + 0.5) / 2 - 0.5 clamped at 0,
    the upper corner clamped at n - 1"""
    U = torch.zeros((2 * n, n), dtype=torch.float64, device=device)
    for o in range(2 * n):
        f = max((o + 0.5) * 0.5 - 0.5, 0.0)
        i0 = int(f)
        i1 = min(i0 + 1, n - 1)
        U[o, i0] += 1.0 - (f - i0)
        U[o, i1] += f - i0
    return U


def upsample2x(x: torch.Tensor) -> dict:
    """stp3_upsample2x_window_f32: x (n_img, h, w, C) -> (n_img, 2h, 2w, C)"""
    _, h, w, _ = x.shape
    Uy, Ux = upsample_matrix(h, x.device), upsample_matrix(w, x.device)
    f = lambda t, a, b: torch.einsum("oi,pj,nijc->nopc", a, b, t)        # noqa: E731
    return {"y": f(_d(x), Uy, Ux), "mag": f(_d(x).abs(), Uy, Ux)}


def upsample2x_bwd(gy: torch.Tensor) -> dict:
    """stp3_upsample2x_window_bwd (the adjoint): gy (n_img, 2h, 2w, C) -> (n_img, h, w, C)"""
    _, H2, W2, _ = gy.shape
    Uy, Ux = upsample_matrix(H2 // 2, gy.device), upsample_matrix(W2 // 2, gy.device)
    f = lambda t: torch.einsum("oi,pj,nopc->nijc", Uy, Ux, t)             # noqa: E731
    return {"gx": f(_d(gy)), "mag": f(_d(gy).abs())}


def phase_interleave(phases: List[Optional[torch.Tensor]], H: int, W: int) -> torch.Tensor:
    """stp3_phase_interleave: phase (py, px) (index 2 py + px) of size (n_img, (H - py + 1) / 2, (W - px + 1) / 2, C)
    or None (zeros) -> (n_img, H, W, C), an exact copy (returned in the phases' dtype)"""
    ref = next(t for t in phases if t is not None)
    out = torch.zeros((ref.shape[0], H, W, ref.shape[-1]), dtype=ref.dtype, device=ref.device)
    for k, t in enumerate(phases):
        if t is not None:
            out[:, k // 2::2, k % 2::2] = t
    return out


def sigmoid_bwd(g: torch.Tensor, s: torch.Tensor) -> dict:
    """stp3_sigmoid_bwd: dz = g s (1 - s)"""
    dz = _d(g) * _d(s) * (1.0 - _d(s))
    return {"dz": dz, "mag": dz.abs()}
