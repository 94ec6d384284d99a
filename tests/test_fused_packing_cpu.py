"""Host logic of the two back-to-back kernels, checked without a GPU: the packed weight blocks, tap tables, chain
descriptors, piece map and bias tables that `DeepLabHead._pack` / `TemporalBlock._pack` hand to stp3_aspp_fused_fwd /
stp3_block_fused_fwd are run through a plain fp64 emulation of what the kernels do with them (the indexing documented in
include/stp3_b200.h and stp3_b200/csrc/{aspp,block}_fused.cu: block order, weight rows of an N-wide chain, K-step ranges,
hidden-accumulator columns, pieces of P) and compared with the fp64 oracle of the same module.  A packing / table mistake shows up here as
an O(1) error; the bf16 hi+lo split of the weights leaves ~1e-5.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import torch_dense as TD  # noqa: E402
from stp3_b200.layers.convolutions import DeepLabHead  # noqa: E402
from stp3_b200.layers.temporal import TemporalBlock  # noqa: E402


def f64(m):
    import copy
    return copy.deepcopy(m).double()


def shifted(x, dt, dy, dx):
    """x (B,T,H,W,C) -> y[b,t,h,w] = x[b,t+dt,h+dy,w+dx] with zeros outside (what a TMA box delivers)."""
    B, T, H, W, C = x.shape
    p = F.pad(x, (0, 0, abs(dx), abs(dx), abs(dy), abs(dy), abs(dt), abs(dt)))
    return p[:, abs(dt) + dt:abs(dt) + dt + T, abs(dy) + dy:abs(dy) + dy + H, abs(dx) + dx:abs(dx) + dx + W]


def blocks_f64(w):
    """(n_blocks, 2, 128, 64) bf16 [hi | lo] -> (n_blocks, 128, 64) fp64"""
    return w[:, 0].double() + w[:, 1].double()


# ----------------------------------------------------------------------------------------------- aspp_fused
def emulate_aspp(x, pa, img_bias, relu=True):
    """aspp_fused.cu: per branch s, acc1 = sum over its taps t and K blocks kb of x[.., kb] . W[t * kblocks + kb]^T (taps
    numbered through all branches); P = relu(acc1 + br_bias[s]); acc2 += P[:, kb2] . W[proj_blk0 + 2 s + kb2]^T;
    y = [relu](acc2 + img_bias[image])."""
    W = blocks_f64(pa.w)
    B, T, H, Wd, cin_p = x.shape
    assert cin_p == pa.cin_p
    kbs = cin_p // 64
    n_taps = sum(len(t) for t in pa.taps)
    proj_blk0 = n_taps * kbs
    assert W.shape[0] == proj_blk0 + 2 * len(pa.taps)
    acc2 = torch.zeros((B, T, H, Wd, 128), dtype=torch.float64)
    t = 0
    for s, taps in enumerate(pa.taps):
        acc1 = torch.zeros((B, T, H, Wd, 128), dtype=torch.float64)
        for (dy, dx) in taps:
            xs = shifted(x, 0, dy, dx)
            for kb in range(kbs):
                acc1 += xs[..., kb * 64:(kb + 1) * 64] @ W[t * kbs + kb].T
            t += 1
        P = torch.relu(acc1 + pa.br_bias[s].double())
        for kb2 in range(2):
            acc2 += P[..., kb2 * 64:(kb2 + 1) * 64] @ W[proj_blk0 + 2 * s + kb2].T
    y = acc2 + img_bias.double().view(B, T, 1, 1, 128)
    return torch.relu(y) if relu else y


@pytest.mark.parametrize("cin,classes,H,W", [(64, 64, 40, 44)])
def test_deeplab_head_fused_packing_vs_oracle(cin, classes, H, W):
    """DeepLabHead(64 -> 64, hidden 128) of the temporal model: ASPP branches + projection (pack 'fused') and the
    3x3 -> classifier tail (pack 'tail', a one-branch instance), emulated from the packed tables, against the oracle."""
    torch.manual_seed(0)
    with torch.no_grad():
        head = TD.init_exact(DeepLabHead(cin, classes, hidden_channel=128), seed=3).eval()
        x = torch.relu(torch.randn(2, cin, H, W)).double()
        ref = TD.deeplab_head(x, f64(head))
        P = head.packed()
        assert "fused" in P and "tail" in P
        xl = x.permute(0, 2, 3, 1).reshape(2, 1, H, W, cin)
        # per-image projection bias exactly as forward_hl builds it: projection bias + W_proj[:, pool] . relu(W1 . mean + b1)
        mean = x.mean(dim=(2, 3))
        pooled = torch.relu(mean @ P["pool_w1"].double().T + P["pool_b1"].double())
        pbias = P["proj"].bias.double()[:128] + pooled @ P["pool_w2"].double().T
        y = emulate_aspp(xl, P["fused"], pbias.view(2, 128))
        tail_bias = P["tail"].proj_bias.double().unsqueeze(0).expand(2, -1)
        z = emulate_aspp(y, P["tail"], tail_bias, relu=False)[..., :classes]
        out = z.reshape(2, H, W, classes).permute(0, 3, 1, 2)
    err = float((out - ref).abs().max() / ref.abs().max())
    print(f"deeplab head from packed tables: {err:.2e} of max")
    assert err < 2e-4


# ----------------------------------------------------------------------------------------------- block_fused
def unpair(blk, n):
    """inverse of dense._pair_rows: rows [0, n/2) and [64, 64 + n/2) of a 128-row block -> the chain's n weight rows"""
    return torch.cat([blk[:n // 2], blk[64:64 + n - n // 2]])


def emulate_block_tail(mid, x, pb, hid_bias, img_bias, res_bias):
    """block_fused.cu: chain c accumulates sum over its taps of src[.., cin_off : cin_off + 64] (shifted) . W_tap^T into
    columns [tmem_col, tmem_col + n_mma) of the hidden accumulator (only K steps [k_lo, k_hi) are issued); piece pp of P =
    relu(acc[piece_col[pp] : +8] + hid_bias[8 pp : +8]) (zeros for -1); out = relu(P . W_agg^T + img_bias) + (x . W_res^T +
    res_bias | x)."""
    W = blocks_f64(pb.w)
    B, T, H, Wd, _ = x.shape
    acc = torch.zeros((B, T, H, Wd, 160), dtype=torch.float64)
    blk = 0
    for src, cin_off, taps, n_mma, tmem_col, k_lo, k_hi in pb.chains:
        assert n_mma % 16 == 0 and tmem_col + n_mma <= 160 and k_lo % 16 == 0 and k_hi % 16 == 0
        inp = (x if src else mid)[..., cin_off:cin_off + 64]
        assert inp.shape[-1] == 64
        for (dt, dy, dx) in taps:
            w = unpair(W[blk], n_mma)
            assert float(w[:, :k_lo].abs().max() if k_lo else 0) == 0 and float(w[:, k_hi:].abs().max() if k_hi < 64 else 0) == 0, \
                "weights outside the issued K steps"
            acc[..., tmem_col:tmem_col + n_mma] += shifted(inp, dt, dy, dx)[..., k_lo:k_hi] @ w[:, k_lo:k_hi].T
            blk += 1
    P = torch.zeros((B, T, H, Wd, 128), dtype=torch.float64)
    hb = hid_bias.double().view(B, T, 1, 1, 128)
    for pp, col in enumerate(pb.piece_col):
        if col >= 0:
            P[..., 8 * pp:8 * pp + 8] = torch.relu(acc[..., col:col + 8] + hb[..., 8 * pp:8 * pp + 8])
    out = torch.zeros((B, T, H, Wd, 64), dtype=torch.float64)
    for kb2 in range(2):
        out += P[..., kb2 * 64:(kb2 + 1) * 64] @ unpair(W[blk], 64).T
        blk += 1
    out = torch.relu(out + img_bias.double().view(B, T, 1, 1, 64))
    if pb.res is not None:
        _, cin_off, _, n_mma, _, k_lo, k_hi = pb.res
        w = unpair(W[blk], n_mma)
        blk += 1
        assert float(w[:, k_hi:].abs().max() if k_hi < 64 else 0) == 0
        out += x[..., cin_off + k_lo:cin_off + k_hi] @ w[:, k_lo:k_hi].T + res_bias.double().view(B, T, 1, 1, 64)
    else:
        out += x[..., :64]
    assert blk == W.shape[0]
    return out


@pytest.mark.parametrize("cin,nc", [(70, 6), (64, 0)])
def test_temporal_block_fused_packing_vs_oracle(cin, nc):
    """Block 1 of the reference (70 -> 64: three 35-channel chains, projection, six ego-motion channels as per-image
    biases) and block 2 (64 -> 64: block-diagonal chain of the two 32-channel paths + path 2, identity residual)."""
    B, T, H, W = 1, 3, 20, 24
    torch.manual_seed(1)
    with torch.no_grad():
        blk = TD.init_exact(TemporalBlock(cin, 64, use_pyramid_pooling=True, pool_sizes=[(2, H, W)]), seed=5).eval()
        blk.n_const = nc
        x = torch.relu(torch.randn(B, cin, T, H, W)).double()
        if nc:
            x[:, cin - nc:] = x[:, cin - nc:, :, :1, :1]            # spatially constant trailing channels
        ref = TD.temporal_block(x, f64(blk))                         # (B, 64, T, H, W)
        P = blk.packed()
        assert "tail" in P
        cs, o, half = P["cs"], P["o"], blk.half_channels
        xl = x.permute(0, 2, 3, 4, 1)                                # (B,T,H,W,cin)
        xs = torch.zeros((B, T, H, W, 64), dtype=torch.float64)
        xs[..., :cs] = xl[..., :cs]
        const = xl[:, :, 0, 0, cs:].reshape(B * T, nc) if nc else None
        # entry convolutions of paths 0 / 1 (a 1x1x1 launch before the fused kernel): mid = relu(W_a1 x + b (+ W_c const))
        wa = torch.zeros(P["nmid"], cs, dtype=torch.float64)
        p0, p1 = blk.convolution_paths[0], blk.convolution_paths[1]
        from stp3_b200 import dense
        w0, b0 = dense.fold_bn(p0[0].conv.weight, p0[0].norm)
        w1, b1 = dense.fold_bn(p1[0].conv.weight, p1[0].norm)
        m1 = P["m1"]
        ba = torch.zeros(P["nmid"], dtype=torch.float64)
        wa[:half], wa[m1:m1 + half] = w0.reshape(half, -1)[:, :cs].double(), w1.reshape(half, -1)[:, :cs].double()
        ba[:half], ba[m1:m1 + half] = b0.double(), b1.double()
        mid_bias = ba.unsqueeze(0).expand(B * T, -1)
        if nc:
            mid_bias = mid_bias + const @ P["a1_c"].double().T
        mid = torch.relu(xs[..., :cs] @ wa.T + mid_bias.view(B, T, 1, 1, -1))
        if mid.shape[-1] < 128:
            mid = F.pad(mid, (0, 128 - mid.shape[-1]))
        # bias tables exactly as _forward_fused builds them
        hid = P["tail_hid_bias"].double().unsqueeze(0).expand(B * T, -1)
        if nc:
            hid = hid + const @ P["tail_hid_c"].double().T
        # aggregation bias + pyramid-pooling branch (reference: temporal.py:408-423 -- mean over a 2-frame causal window)
        pooled = TD.pyramid_pooling(x, f64(blk).pyramid_pooling)[:, :, :, 0, 0]           # (B, n_pool, T), constant over H, W
        wg, bg = dense.fold_bn(blk.aggregation[0].conv.weight, blk.aggregation[0].norm)
        wg = wg.reshape(wg.shape[0], -1).double()
        pbias = bg.double().view(1, 1, -1) + pooled.permute(0, 2, 1) @ wg[:, 3 * half:].T   # (B, T, 64)
        rbias = None
        if blk.projection is not None:
            wj, bj = dense.fold_bn(blk.projection[0].weight, blk.projection[1])
            wj = wj.reshape(wj.shape[0], -1).double()
            rbias = bj.double().unsqueeze(0).expand(B * T, -1)
            if nc:
                rbias = rbias + const @ wj[:, cs:].T
        out = emulate_block_tail(mid, xs, P["tail"], hid.reshape(B * T, 128), pbias.reshape(B * T, 64),
                                 None if rbias is None else rbias.reshape(B * T, 64))
    got = out.permute(0, 4, 1, 2, 3)
    err = float((got - ref).abs().max() / ref.abs().max())
    print(f"temporal block {cin}->64 from packed tables: {err:.2e} of max")
    assert err < 2e-4
