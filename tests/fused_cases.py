"""Synthetic descriptors of the two back-to-back kernels (stp3_aspp_fused_fwd, stp3_block_fused_fwd), built through
dense.pack_aspp / dense.pack_block_tail from random weights, with the raw weights kept for a direct F.conv2d / F.conv3d
composition.  Weights are bf16 values (their packed lo plane is zero), so the fp64 reference of the packed tables and
the composition agree to rounding.  Used by tests/test_fused_reference_cpu.py and tests/test_fused_contract_gpu.py."""
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

from stp3_b200 import dense


def rnd(*shape, seed: int, scale: float = 1.0, dev="cpu") -> torch.Tensor:
    """uniform in [-scale, scale), rounded to bf16 (exact in the packed hi plane), fp32"""
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(*shape, generator=g) * 2 - 1) * scale).to(torch.bfloat16).float().to(dev)


def planes(B, T, H, W, c, cs, seed, dev="cpu") -> dense.HL:
    """(B, T, H, W, cs) hi/lo planes: channels [0, c) random fp32 values, channels [c, cs) large values no kernel
    may read (a read shows up as an O(100) error)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, T, H, W, cs, generator=g) * 2 - 1
    x[..., c:] = 100.0 + x[..., c:]
    hi, lo = dense.split_hilo(x.to(dev))
    return dense.HL(hi, lo, c)


# ----------------------------------------------------------------------------------------------- aspp
@dataclass
class AsppCase:
    pa: dense.PackedAspp
    branches: List[Tuple[torch.Tensor, torch.Tensor, Tuple[int, int]]]   # (w (128, cin, k, k), b (128), (ry, rx))
    proj_w: torch.Tensor                                                 # (128, n_br * 128), zero rows past n_out
    cin: int


def aspp_case(cin: int, rates, n_out: int = 128, seed: int = 0, dev="cpu") -> AsppCase:
    """rates: per branch None (a 1x1 branch) or (ry, rx) (a 3x3 branch with taps (iy - 1) ry, (ix - 1) rx)."""
    br, raw = [], []
    for i, r in enumerate(rates):
        k = 1 if r is None else 3
        w = rnd(128, cin, k, k, seed=seed + 10 * i + 1, scale=1.5 / (cin * k * k) ** 0.5, dev=dev)
        b = rnd(128, seed=seed + 10 * i + 2, scale=0.3, dev=dev)
        br.append((w, b, 1))
        raw.append((w, b, (0, 0) if r is None else tuple(r)))
    pw = rnd(n_out, 128 * len(rates), seed=seed + 7, scale=2.0 / (128 * len(rates)) ** 0.5, dev=dev)
    pb = rnd(n_out, seed=seed + 8, scale=0.2, dev=dev)
    pa = dense.pack_aspp(br, pw, pb)
    # the tap offsets of each branch at its own vertical / horizontal rate (the weight blocks do not depend on them)
    pa.taps = [[(0, 0)] if r is None else [((iy - 1) * r[0], (ix - 1) * r[1]) for iy in range(3) for ix in range(3)]
               for r in rates]
    proj = torch.zeros(128, 128 * len(rates), device=dev)
    proj[:n_out] = pw
    return AsppCase(pa, raw, proj, cin)


def aspp_direct(case: AsppCase, x: torch.Tensor, img_bias: torch.Tensor, relu: bool = True) -> torch.Tensor:
    """The same operation as F.conv2d calls: x (n_img, cin, H, W) float64 -> (n_img, H, W, 128)"""
    P = []
    for w, b, (ry, rx) in case.branches:
        pad = (ry, rx) if w.shape[-1] == 3 else (0, 0)
        y = F.conv2d(x, w.double(), b.double(), padding=pad, dilation=(max(ry, 1), max(rx, 1)))
        P.append(torch.relu(y))
    y = torch.cat(P, 1).permute(0, 2, 3, 1) @ case.proj_w.double().t() + img_bias.double().view(-1, 1, 1, 128)
    return torch.relu(y) if relu else y


# ----------------------------------------------------------------------------------------------- block
@dataclass
class BlockCase:
    pb: dense.PackedBlockTail
    chains: list                      # (src, cin_off, w (cout, cin, kt, kh, kw), k_off, n_mma, tmem_col)
    agg_w: torch.Tensor               # (64, 128) in P order
    res_w: Optional[torch.Tensor]     # (64, cs)
    cs: int
    layout: int                       # 0 = three paths, 1 = block-diagonal pair


def block_case(layout: int, proj: bool, cs: int = 64, seed: int = 0, dev="cpu") -> BlockCase:
    """The two chain layouts the kernel is compiled for, as TemporalBlock._pack builds them:
      0: three 35-channel paths at N = 48 (causal (2,3,3) of mid[0:35], (1,3,3) of mid[64:99], 1x1x1 of x[0:cs]);
      1: a (2,3,3) chain of all 64 mid channels at N = 64, then a 32-channel 1x1x1 of x at N = 32."""
    def w(cout, cin, kt, kh, kw, s):
        return rnd(cout, cin, kt, kh, kw, seed=seed + s, scale=1.5 / (cin * kt * kh * kw) ** 0.5, dev=dev)
    if layout == 0:
        half, n16, o = 35, 48, 40
        chains = [(0, 0, w(half, half, 2, 3, 3, 1), 0, n16, 0), (0, 64, w(half, half, 1, 3, 3, 2), 0, n16, n16),
                  (1, 0, w(half, cs, 1, 1, 1, 3), 0, n16, 2 * n16)]
        piece_col = [n16 * k + 8 * q for k in range(3) for q in range(o // 8)]
    else:
        chains = [(0, 0, w(64, 64, 2, 3, 3, 1), 0, 64, 0), (1, 0, w(32, cs, 1, 1, 1, 3), 0, 32, 64)]
        piece_col = [8 * pp for pp in range(8)] + [64 + 8 * q for q in range(4)]
    piece_col += [-1] * (16 - len(piece_col))
    agg_w = rnd(64, 128, seed=seed + 5, scale=2.0 / 128 ** 0.5, dev=dev)
    res_w = rnd(64, cs, seed=seed + 6, scale=1.0 / cs ** 0.5, dev=dev) if proj else None
    pb = dense.pack_block_tail(chains, agg_w, res_w, piece_col)
    return BlockCase(pb, chains, agg_w, res_w, cs, layout)


def block_direct(case: BlockCase, mid: torch.Tensor, x: torch.Tensor, hid_bias, img_bias, res_bias):
    """The same operation as F.conv3d calls: mid, x (B, C, T, H, W) float64 -> (B*T, H, W, 64)"""
    B, _, T, H, W = x.shape
    hidden = x.new_zeros((B, 160, T, H, W))
    for src, cin_off, w, k_off, n_mma, tmem_col in case.chains:
        cout, cin, kt, kh, kw = w.shape
        inp = (x if src else mid)[:, cin_off + k_off:cin_off + k_off + cin]
        inp = F.pad(inp, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
        hidden[:, tmem_col:tmem_col + cout] = F.conv3d(inp, w.double())
    P = x.new_zeros((B, 128, T, H, W))
    hb = hid_bias.double().view(B, T, 128).permute(0, 2, 1)[..., None, None]
    for pp, col in enumerate(case.pb.piece_col):
        if col >= 0:
            P[:, 8 * pp:8 * pp + 8] = torch.relu(hidden[:, col:col + 8] + hb[:, 8 * pp:8 * pp + 8])
    P = P.permute(0, 2, 3, 4, 1)
    out = torch.relu(P @ case.agg_w.double().t() + img_bias.double().view(B, T, 1, 1, 64))
    xl = x.permute(0, 2, 3, 4, 1)
    if case.res_w is not None:
        out = out + xl[..., :case.cs] @ case.res_w.double().t() + res_bias.double().view(B, T, 1, 1, 64)
    else:
        out = out + xl[..., :64]
    return out.reshape(B * T, H, W, 64)
