"""Float64 reference of the two back-to-back kernels' contracts, stp3_aspp_fused_fwd and stp3_block_fused_fwd
(include/stp3_b200.h), evaluated from the stored bf16 input planes, the packed weight blocks (w[:, 0] hi, w[:, 1] lo) and
the descriptor fields rather than from a PyTorch layer.  Runs on CPU or CUDA tensors (float64 matmuls only; on the
device that is DGEMM, which uses no TF32), like tests/conv_reference.py does for stp3_conv_fwd.

Both kernels chain two products: a first MMA chain into a register accumulator, its activated output P split to bf16
hi/lo in registers, and P fed back as the A operand of a second chain.

  exact:  (x_hi + x_lo) . (w_hi + w_lo) in both stages, P = relu(acc1 + bias) unsplit: the operation the planes and the
          packed weights describe
  model:  the products the kernel issues: stage 1 = x_hi.w_hi + x_hi.w_lo + x_lo.w_hi; P split as ptx::split_hilo does
          it (hi = bf16(p), lo = bf16(p - hi)); stage 2 = P_hi.W_hi + P_hi.W_lo + P_lo.W_hi.  The block's projection
          acc3 is a stage-1 product of x.

The identity residual of the block adds x_hi + x_lo in both modes.  The aspp reference returns the n_store stored
channels; the block reference returns the 64 output channels and the per-image column sums over in-image pixels of the
output before its hi/lo split.
"""
from typing import Optional, Tuple

import torch

from stp3_b200 import dense


def split(p: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """ptx::split_hilo of the fp32 value of p: hi = bf16(p), lo = bf16(p - hi), both returned as float64."""
    p32 = p.float()
    hi = p32.to(torch.bfloat16)
    lo = (p32 - hi.float()).to(torch.bfloat16)
    return hi.double(), lo.double()


def shifted(x: torch.Tensor, dt: int, dy: int, dx: int) -> torch.Tensor:
    """x (B, T, H, W, C) -> y[b, t, h, w] = x[b, t + dt, h + dy, w + dx], zero outside the tensor (what a TMA box of
    the tap delivers; offsets beyond the map give all zeros)."""
    B, T, H, W, C = x.shape
    out = x.new_zeros(x.shape)
    t0, t1 = max(0, -dt), min(T, T - dt)
    y0, y1 = max(0, -dy), min(H, H - dy)
    x0, x1 = max(0, -dx), min(W, W - dx)
    if t0 < t1 and y0 < y1 and x0 < x1:
        out[:, t0:t1, y0:y1, x0:x1] = x[:, t0 + dt:t1 + dt, y0 + dy:y1 + dy, x0 + dx:x1 + dx]
    return out


def _product(a_hi, a_lo, w_hi, w_lo, model: bool) -> torch.Tensor:
    """a (..., K) . w (N, K)^T: exact (a_hi + a_lo) . (w_hi + w_lo) or the kernel's three products"""
    if model:
        return a_hi @ w_hi.t() + a_hi @ w_lo.t() + a_lo @ w_hi.t()
    return (a_hi + a_lo) @ (w_hi + w_lo).t()


def _stage2(p: torch.Tensor, w_hi, w_lo, model: bool) -> torch.Tensor:
    """P . W^T with P from registers: unsplit (exact) or split into hi / lo and multiplied with three products (model)"""
    if model:
        p_hi, p_lo = split(p)
        return _product(p_hi, p_lo, w_hi, w_lo, True)
    return p @ (w_hi + w_lo).t()


def _weights(w: torch.Tensor, dev) -> Tuple[torch.Tensor, torch.Tensor]:
    """(n_blocks, 2, 128, 64) bf16 [hi | lo] -> two (n_blocks, 128, 64) float64 tensors on dev"""
    return w[:, 0].double().to(dev), w[:, 1].double().to(dev)


# ----------------------------------------------------------------------------------------------- aspp_fused
def aspp(x_hi: torch.Tensor, x_lo: torch.Tensor, pa: dense.PackedAspp, img_bias: torch.Tensor, *, n_store: int = 128,
         relu: bool = True, model: bool = False) -> torch.Tensor:
    """stp3_aspp_fused_fwd: x planes (B, T, H, W, in_cstride), channels [0, pa.cin_p) read.  Per branch s: acc1 = sum
    over its taps t (numbered through all branches) and K blocks kb of x[.., kb] . W[t * kblocks + kb]^T;
    P = relu(acc1 + br_bias[s]); acc2 += P[:, kb2] . W[proj_blk0 + 2 s + kb2]^T.  Returns [relu](acc2 + img_bias[image])
    channels [0, n_store) as (B*T, H, W, n_store) float64."""
    B, T, H, W, cs = x_hi.shape
    dev = x_hi.device
    cin = pa.cin_p
    assert cin % 64 == 0 and cin <= cs
    kbs = cin // 64
    wh, wl = _weights(pa.w, dev)
    n_taps = sum(len(t) for t in pa.taps)
    proj_blk0 = n_taps * kbs
    assert wh.shape[0] == proj_blk0 + 2 * len(pa.taps)
    xh, xl = x_hi[..., :cin].double(), x_lo[..., :cin].double()
    br_bias = pa.br_bias.double().to(dev)
    acc2 = xh.new_zeros((B, T, H, W, 128))
    t = 0
    for s, taps in enumerate(pa.taps):
        acc1 = xh.new_zeros((B, T, H, W, 128))
        for (dy, dx) in taps:
            ah, al = shifted(xh, 0, dy, dx), shifted(xl, 0, dy, dx)
            for kb in range(kbs):
                k = slice(kb * 64, (kb + 1) * 64)
                acc1 += _product(ah[..., k], al[..., k], wh[t * kbs + kb], wl[t * kbs + kb], model)
            t += 1
        P = torch.relu(acc1 + br_bias[s])
        del acc1
        for kb2 in range(2):
            blk = proj_blk0 + 2 * s + kb2
            acc2 += _stage2(P[..., kb2 * 64:(kb2 + 1) * 64], wh[blk], wl[blk], model)
    y = acc2 + img_bias.double().to(dev).view(B, T, 1, 1, 128)
    if relu:
        y = torch.relu(y)
    return y[..., :n_store].reshape(B * T, H, W, n_store)


# ----------------------------------------------------------------------------------------------- block_fused
def unpair(blk: torch.Tensor, n: int) -> torch.Tensor:
    """inverse of dense._pair_rows: rows [0, n/2) and [64, 64 + n/2) of a 128-row block -> the chain's n weight rows"""
    return torch.cat([blk[:n // 2], blk[64:64 + n - n // 2]])


def block_tail(mid_hi: torch.Tensor, mid_lo: torch.Tensor, x_hi: torch.Tensor, x_lo: torch.Tensor,
               pb: dense.PackedBlockTail, hid_bias: torch.Tensor, img_bias: torch.Tensor,
               res_bias: Optional[torch.Tensor], *, model: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """stp3_block_fused_fwd: chain c accumulates, over its taps, src[.., cin_off + k_lo : cin_off + k_hi] (shifted)
    times the tap's weights into hidden columns [tmem_col, tmem_col + n_mma); piece pp of P = relu(acc[piece_col[pp] : +8]
    + hid_bias[8 pp : +8]) (zeros for -1); out = relu(P . W_agg^T + img_bias) + (x . W_res^T + res_bias | x).
    Returns (out (B*T, H, W, 64), col_sums (B*T, 64)) in float64."""
    B, T, H, W, _ = x_hi.shape
    dev = x_hi.device
    n_img = B * T
    wh, wl = _weights(pb.w, dev)
    planes = {0: (mid_hi.double(), mid_lo.double()), 1: (x_hi.double(), x_lo.double())}
    acc = planes[1][0].new_zeros((B, T, H, W, 160))
    blk = 0
    last_src = None
    for src, cin_off, taps, n_mma, tmem_col, k_lo, k_hi in pb.chains:
        assert n_mma % 16 == 0 and tmem_col + n_mma <= 160 and k_lo % 16 == 0 and k_hi % 16 == 0 and k_lo < k_hi <= 64
        ph, pl = (p[..., cin_off + k_lo:cin_off + k_hi] for p in planes[src])
        for (dt, dy, dx) in taps:
            w_hi, w_lo = unpair(wh[blk], n_mma)[:, k_lo:k_hi], unpair(wl[blk], n_mma)[:, k_lo:k_hi]
            acc[..., tmem_col:tmem_col + n_mma] += _product(shifted(ph, dt, dy, dx), shifted(pl, dt, dy, dx),
                                                             w_hi, w_lo, model)
            blk += 1
        last_src = (src, cin_off)
    P = acc.new_zeros((B, T, H, W, 128))
    hb = hid_bias.double().to(dev).view(B, T, 1, 1, 128)
    for pp, col in enumerate(pb.piece_col):
        if col >= 0:
            P[..., 8 * pp:8 * pp + 8] = torch.relu(acc[..., col:col + 8] + hb[..., 8 * pp:8 * pp + 8])
    del acc
    out = P.new_zeros((B, T, H, W, 64))
    for kb2 in range(2):
        out += _stage2(P[..., kb2 * 64:(kb2 + 1) * 64], unpair(wh[blk], 64), unpair(wl[blk], 64), model)
        blk += 1
    out = torch.relu(out + img_bias.double().to(dev).view(B, T, 1, 1, 64))
    if pb.res is not None:
        _, cin_off, _, n_mma, _, k_lo, k_hi = pb.res
        assert last_src == (1, cin_off), "the projection reads the last chain's activations: x at the same K block"
        w_hi, w_lo = unpair(wh[blk], n_mma)[:, k_lo:k_hi], unpair(wl[blk], n_mma)[:, k_lo:k_hi]
        blk += 1
        xh, xl = (p[..., cin_off + k_lo:cin_off + k_hi] for p in planes[1])
        out += _product(xh, xl, w_hi, w_lo, model) + res_bias.double().to(dev).view(B, T, 1, 1, 64)
    else:
        out += planes[1][0][..., :64] + planes[1][1][..., :64]
    assert blk == wh.shape[0]
    out = out.reshape(n_img, H, W, 64)
    return out, out.sum(dim=(1, 2))
