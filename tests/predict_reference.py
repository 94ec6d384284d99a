"""float64 reference of the prediction stage's per-pixel kernels (csrc/predict_kernels.cu, include/stp3_b200.h):
stp3_gru_gates, stp3_gru_update, stp3_channel_norm_act, stp3_dw_ln, stp3_trust_mix, stp3_maxpool2_pad (bit-exact),
stp3_hl_copy (bit-exact) and stp3_hl_broadcast (bit-exact: the hi/lo split of the fp32 vector).

Every function takes the values of one call's slots, channels last (..., C) in float64 (hi + lo of the stored planes),
with the fp32 parameters as they are, and returns the value `y` of every written element and `mag`, the sum of the
magnitudes of the terms that make up each value: the scale a fixed-order fp32 evaluation's round-off grows with.
  - gru_gates: |h|.  1 - sigmoid(r) cancels as r grows, so its fp32 error is an absolute 2^-24, not a relative one.
  - gru_update: |h| + |h_tilde|.
  - LayerNorm: (|a| + mean |a|) inv |gamma| + |beta|, a the normalised vector (x for stp3_channel_norm_act, the
    depthwise output for stp3_dw_ln) and inv = 1 / sqrt(var + eps).  mean |a| is the magnitude of the mean's terms, so
    a mean of 1e3 over a spread of 1e-2 is held to what fp32 can resolve; for stp3_dw_ln every |a| is replaced by the
    tap magnitudes sum |w| |x| + |b|.
  - GELU: the magnitude of its argument (|gelu(v)| <= |v| and |gelu'| <= 1.13); an added y (or gelu(y)): + |y|.
  - trust_mix: |s2| p0 + |s1| p1 + |s1 - s2| p0 p1 sum_k sum_c |w_kc| |t_c|: the logits' round-off moves p by p0 p1
    times their own error."""
import math
from typing import Optional, Tuple

import torch

from tests.aux_reference import F64, f32, split  # noqa: F401  (split: the stored hi/lo of an fp32 value)


def planes(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    return hi.to(F64) + lo.to(F64)


def gelu(v: torch.Tensor) -> torch.Tensor:
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def gru_gates(r: torch.Tensor, h: torch.Tensor) -> dict:
    """out = (1 - sigmoid(r)) h"""
    return {"y": (1.0 - torch.sigmoid(r)) * h, "mag": h.abs()}


def gru_update(u: torch.Tensor, h: torch.Tensor, ht: torch.Tensor) -> dict:
    """out = (1 - s) h + s h_tilde, s = sigmoid(u)"""
    s = torch.sigmoid(u)
    return {"y": (1.0 - s) * h + s * ht, "mag": h.abs() + ht.abs()}


def layer_norm(a: torch.Tensor, amag: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> dict:
    """LayerNorm over the last dimension, biased variance; amag the magnitudes of a's own terms"""
    g, b = gamma.to(F64).to(a.device), beta.to(F64).to(a.device)
    mu = a.mean(-1, keepdim=True)
    inv = 1.0 / torch.sqrt(((a - mu) ** 2).mean(-1, keepdim=True) + f32(eps))
    return {"y": (a - mu) * inv * g + b, "mag": (amag + amag.mean(-1, keepdim=True)) * inv * g.abs() + b.abs()}


def channel_norm_act(x: torch.Tensor, ln: Optional[Tuple[torch.Tensor, torch.Tensor, float]] = None, act: bool = False,
                     y: Optional[torch.Tensor] = None, gelu_y: bool = False) -> dict:
    """out = [gelu]([LN](x)) + [gelu](y)"""
    r = layer_norm(x, x.abs(), *ln) if ln is not None else {"y": x, "mag": x.abs()}
    v, mag = r["y"], r["mag"]
    if act:
        v = gelu(v)
    if y is not None:
        v = v + (gelu(y) if gelu_y else y)
        mag = mag + y.abs()
    return {"y": v, "mag": mag}


def depthwise(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """x (N, H, W, C), w (k*k, C) (tap ky * k + kx), zero padding k // 2 -> (sum w x + b, sum |w| |x| + |b|)"""
    N, H, W, C = x.shape
    p = k // 2
    xp = x.new_zeros((N, H + 2 * p, W + 2 * p, C))
    xp[:, p:p + H, p:p + W] = x
    w64, b64 = w.to(F64).to(x.device), b.to(F64).to(x.device)
    acc, mag = b64.expand(N, H, W, C).clone(), b64.abs().expand(N, H, W, C).clone()
    for ky in range(k):
        for kx in range(k):
            t = xp[:, ky:ky + H, kx:kx + W]
            acc += t * w64[ky * k + kx]
            mag += t.abs() * w64[ky * k + kx].abs()
    return acc, mag


def dw_ln(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, k: int, gamma: torch.Tensor, beta: torch.Tensor,
          eps: float) -> dict:
    """out = LN(depthwise k x k (x) + b)"""
    a, amag = depthwise(x, w, b, k)
    return layer_norm(a, amag, gamma, beta, eps)


def trust_mix(t: torch.Tensor, w: torch.Tensor, s1: torch.Tensor, s2: torch.Tensor) -> dict:
    """p = softmax(W t) over the two rows of w (2, C); out = s2 p0 + s1 p1"""
    w64 = w.to(F64).to(t.device)
    z = torch.einsum("kc,...c->...k", w64, t)
    p = torch.softmax(z, -1)
    p0, p1 = p[..., :1], p[..., 1:]
    zmag = torch.einsum("kc,...c->...", w64.abs(), t.abs()).unsqueeze(-1)
    return {"y": s2 * p0 + s1 * p1, "mag": s2.abs() * p0 + s1.abs() * p1 + (s1 - s2).abs() * p0 * p1 * zmag, "p": p}


def maxpool2_pad(hi: torch.Tensor, lo: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(N, H, W, C) planes -> (N, ceil(H/2), ceil(W/2), C): an odd H / W padded by one +0 / +0 row / column, the first
    of the four window elements (row-major) whose fp32 hi + lo no later one exceeds, its planes' bits as stored"""
    N, H, W, C = hi.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    ph, pl = (t.new_zeros((N, 2 * Ho, 2 * Wo, C)) for t in (hi, lo))
    ph[:, :H, :W], pl[:, :H, :W] = hi, lo
    best_h, best_l = ph[:, 0::2, 0::2].clone(), pl[:, 0::2, 0::2].clone()
    m = best_h.float() + best_l.float()
    for dy, dx in ((0, 1), (1, 0), (1, 1)):
        vh, vl = ph[:, dy::2, dx::2], pl[:, dy::2, dx::2]
        v = vh.float() + vl.float()
        take = v > m
        best_h, best_l, m = torch.where(take, vh, best_h), torch.where(take, vl, best_l), torch.where(take, v, m)
    return best_h, best_l
