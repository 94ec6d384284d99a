"""3-D spatio-temporal block with the reference's constructor signatures and parameter names
(stp3/layers/temporal.py:252-273, 315-325, 375-489); forward() runs on the wgmma implicit-GEMM kernels.

TemporalBlock data flow on the device (channels-last hi/lo planes, o = half rounded up to 8):
    x --1x1x1 (paths 0,1 fused, N=128)--> mid[0:half | 64:64+half]
    mid[0:64]  --causal (2,3,3)--> agg[0:o]         mid[64:128] --(1,3,3)--> agg[o:2o]
    x --1x1x1 (path 2)--> agg[2o:3o]
    pyramid pooling (spatially constant, temporal.py:408-423)  -> per-image bias of the aggregation conv
    out = relu(BN(1x1x1(agg))) + (projection(x) | x)
Spatially constant input channels (the broadcast ego-motion of stp3.py:145-152) are never materialised: they enter
every 1x1x1 convolution that reads x as a per-image bias.
"""
import os
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn

from .. import dense
from ._packing import PackedModule


def conv_1x1x1_norm_activated(in_channels, out_channels):
    """1x1x1 Conv3d (no bias) + BatchNorm3d + ReLU, named conv / norm / activation as in the reference."""
    return nn.Sequential(OrderedDict(conv=nn.Conv3d(in_channels, out_channels, kernel_size=1, bias=False),
                                     norm=nn.BatchNorm3d(out_channels), activation=nn.ReLU(inplace=True)))


class CausalConv3d(nn.Module):
    """Parameter container of the causal 3-D convolution (time padded on the left only)."""

    def __init__(self, in_channels, out_channels, kernel_size=(2, 3, 3), dilation=(1, 1, 1), bias=False):
        super().__init__()
        assert len(kernel_size) == 3, 'kernel_size must be a 3-tuple.'
        assert tuple(dilation) == (1, 1, 1), "the reference never dilates its causal convolutions"
        kt, kh, kw = kernel_size
        self.pad = nn.ConstantPad3d(padding=((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0), value=0)
        self.conv = nn.Conv3d(in_channels, out_channels, kernel_size, dilation=dilation, stride=1, padding=0, bias=bias)
        self.norm = nn.BatchNorm3d(out_channels)
        self.activation = nn.ReLU(inplace=True)


class PyramidSpatioTemporalPooling(nn.Module):
    """Parameter container; pool_sizes must be [(2, h, w)] with (h, w) the full map (the reference's only use),
    which makes the branch spatially constant."""

    def __init__(self, in_channels, reduction_channels, pool_sizes):
        super().__init__()
        feats = []
        for pool_size in pool_sizes:
            assert pool_size[0] == 2, "Time kernel should be 2 (as in the reference)"
            feats.append(nn.Sequential(OrderedDict(
                avgpool=nn.AvgPool3d(kernel_size=pool_size, stride=(1, *pool_size[1:]), padding=(pool_size[0] - 1, 0, 0),
                                     count_include_pad=False),
                conv_bn_relu=conv_1x1x1_norm_activated(in_channels, reduction_channels))))
        self.features = nn.ModuleList(feats)
        self.pool_sizes = [tuple(p) for p in pool_sizes]


def _round8(n):
    return (n + 7) // 8 * 8


class TemporalBlock(PackedModule):
    def __init__(self, in_channels, out_channels=None, use_pyramid_pooling=False, pool_sizes=None):
        super().__init__()
        self.in_channels = in_channels
        self.half_channels = in_channels // 2
        self.out_channels = out_channels or self.in_channels
        self.kernels = [(2, 3, 3), (1, 3, 3)]
        self.use_pyramid_pooling = use_pyramid_pooling

        paths = [nn.Sequential(conv_1x1x1_norm_activated(self.in_channels, self.half_channels),
                               CausalConv3d(self.half_channels, self.half_channels, kernel_size=k))
                 for k in self.kernels]
        paths.append(conv_1x1x1_norm_activated(self.in_channels, self.half_channels))
        self.convolution_paths = nn.ModuleList(paths)
        agg_in_channels = len(self.convolution_paths) * self.half_channels

        if self.use_pyramid_pooling:
            assert pool_sizes is not None, "setting must contain the list of kernel_size, but is None."
            assert len(pool_sizes) == 1, "one full-map pool size, as in the reference (temporal_model.py:24)"
            reduction_channels = self.in_channels // 3
            self.pyramid_pooling = PyramidSpatioTemporalPooling(self.in_channels, reduction_channels, pool_sizes)
            agg_in_channels += len(pool_sizes) * reduction_channels

        self.aggregation = nn.Sequential(conv_1x1x1_norm_activated(agg_in_channels, self.out_channels),)

        if self.out_channels != self.in_channels:
            self.projection = nn.Sequential(
                nn.Conv3d(self.in_channels, self.out_channels, kernel_size=1, bias=False),
                nn.BatchNorm3d(self.out_channels),
            )
        else:
            self.projection = None
        self.n_const = 0      # trailing input channels that are spatially constant (set by STP3 for the ego-motion)

    # ------------------------------------------------------------------------------------------------
    def _pack(self):
        cin, half, cout, nc = self.in_channels, self.half_channels, self.out_channels, self.n_const
        cs = cin - nc                                  # spatial input channels
        o = _round8(half)
        assert half <= 128 and cout <= 256, "at most 256 input / output channels per block"
        hp = dense.pad_to(half)                        # channel window of one mid path (multiple of 64)
        ap = dense.pad_to(3 * o)                       # channels of the concat tensor the aggregation conv reads
        P = {"o": o, "cs": cs, "hp": hp, "ap": ap}
        flat = lambda w: w.reshape(w.shape[0], w.shape[1])

        def pad_rows(w, rows):                     # zero rows for the padded output columns: a bias table is written whole
            out = torch.zeros(rows, w.shape[1], device=w.device)
            out[:w.shape[0]] = w
            return out
        p0, p1, p2 = self.convolution_paths
        # fused entry convolutions of paths 0 and 1 (N = 128: path 0 at rows 0.., path 1 at rows 64..)
        w0, b0 = dense.fold_bn(p0[0].conv.weight, p0[0].norm)
        w1, b1 = dense.fold_bn(p1[0].conv.weight, p1[0].norm)
        # path 0 lives at channel 0 of `mid`; path 1 right behind it when both fit one 64-channel K block (block 2 of
        # the reference: 32 + 32), else in the next block (block 1: 35 + 35)
        shared = 2 * half <= 64                        # both mid paths fit one 64-channel K block
        m1 = half if shared else hp
        nmid = 64 if shared else 2 * hp
        P["m1"], P["nmid"] = m1, nmid
        wa = torch.zeros(nmid, cin, device=w0.device)
        ba = torch.zeros(nmid, device=w0.device)
        wa[:half], wa[m1:m1 + half] = flat(w0), flat(w1)
        ba[:half], ba[m1:m1 + half] = b0, b1
        P["a1"] = dense.pack_conv(wa[:, :cs].reshape(nmid, cs, 1, 1).contiguous(), ba, bn=nmid)
        w2, b2 = dense.fold_bn(p2.conv.weight, p2.norm)
        P["a2"] = dense.pack_conv(flat(w2)[:, :cs].reshape(half, cs, 1, 1).contiguous(), b2)
        wt, bt = dense.fold_bn(p0[1].conv.weight, p0[1].norm)          # (half, half, 2, 3, 3)
        P["b"] = dense.pack_conv(wt, bt, cin_p=hp)
        ws, bs = dense.fold_bn(p1[1].conv.weight, p1[1].norm)          # (half, half, 1, 3, 3)
        P["c"] = dense.pack_conv(ws, bs, cin_p=hp, in_layout=[(0, half, m1 % 64)])
        if shared and o + half <= 64:
            # both mid paths live in ONE 64-channel block (block 2 of the reference: 32 + 32): the causal (2,3,3) and the
            # (1,3,3) convolution run as one block-diagonal launch -- every activation tile is fetched once instead of
            # twice (these layers are bound by the L2 -> SM traffic of their shifted windows, not by the MMAs), the
            # zero off-diagonal blocks cost tensor work that is free here
            kt = wt.shape[2]
            wbc = torch.zeros(o + half, 64, kt, 3, 3, device=wt.device)
            bbc = torch.zeros(o + half, device=wt.device)
            wbc[:half, :half] = wt
            wbc[o:o + half, m1:m1 + half, kt - 1] = ws[:, :, 0]          # the (1,3,3) kernel sees the present frame only
            bbc[:half], bbc[o:o + half] = bt, bs
            P["bc"] = dense.pack_conv(wbc, bbc, cin_p=64, bn=64)
        wg, bg = dense.fold_bn(self.aggregation[0].conv.weight, self.aggregation[0].norm)
        wg = flat(wg)
        P["agg"] = dense.pack_conv(wg[:, :3 * half].reshape(cout, 3 * half, 1, 1).contiguous(), bg,
                                   in_layout=[(0, half, 0), (half, half, o), (2 * half, half, 2 * o)], cin_p=ap)
        if self.use_pyramid_pooling:
            wp, bp = dense.fold_bn(self.pyramid_pooling.features[0].conv_bn_relu.conv.weight,
                                   self.pyramid_pooling.features[0].conv_bn_relu.norm)
            P["pool_w1"], P["pool_b1"] = flat(wp).contiguous(), bp.contiguous()
            P["pool_w2"] = pad_rows(wg[:, 3 * half:], P["agg"].bn)
        if self.projection is not None:
            wj, bj = dense.fold_bn(self.projection[0].weight, self.projection[1])
            P["proj"] = dense.pack_conv(flat(wj)[:, :cs].reshape(cout, cs, 1, 1).contiguous(), bj)
            P["proj_c"] = pad_rows(flat(wj)[:, cs:], P["proj"].bn)
        if nc:
            P["a1_c"] = wa[:, cs:].contiguous()
            P["a2_c"] = pad_rows(flat(w2)[:, cs:], P["a2"].bn)
        # Two 64-column 1x1x1 convolutions of x as ONE 128-column launch with two destinations (x is read once):
        #   no projection (block 2 of the reference): [paths 0+1 entry -> mid | path 2 -> concat tensor]
        #   projection   (block 1):                    [path 2 -> concat tensor | projection -> skip tensor]
        w2p, b2p = pad_rows(flat(w2), 64) if half <= 64 else None, None
        if half <= 64:
            b2p = torch.zeros(64, device=w0.device); b2p[:half] = b2
        if self.projection is None and nmid == 64 and half <= 64:
            wm = torch.cat([wa, w2p], 0)
            P["a12"] = dense.pack_conv(wm[:, :cs].reshape(128, cs, 1, 1).contiguous(), torch.cat([ba, b2p]), bn=128)
            if nc:
                P["a12_c"] = wm[:, cs:].contiguous()
        if self.projection is not None and half <= 64 and cout <= 64:
            wjp = pad_rows(flat(wj), 64)
            bjp = torch.zeros(64, device=w0.device); bjp[:cout] = bj
            wm = torch.cat([w2p, wjp], 0)
            P["a2p"] = dense.pack_conv(wm[:, :cs].reshape(128, cs, 1, 1).contiguous(), torch.cat([b2p, bjp]), bn=128)
            if nc:
                P["a2p_c"] = wm[:, cs:].contiguous()
        # ---- the block's tail as ONE back-to-back kernel (stp3_block_fused_fwd): paths + aggregation + residual
        n16 = (half + 15) // 16 * 16
        if (os.environ.get("STP3_BLOCK_FUSED", "1") != "0" and cout <= 64 and cs <= 64 and hp == 64 and 3 * o <= 128 and
                3 * n16 <= 144 and (not shared or 2 * o == 64)):
            w2r = flat(w2)[:, :cs].reshape(half, cs, 1, 1, 1)
            if shared:       # both mid paths in one K block: one block-diagonal chain, then path 2
                chains = [(0, 0, wbc, 0, 64, 0), (1, 0, w2r, 0, n16, 64)]
                piece_col = [8 * pp for pp in range(8)] + [64 + 8 * q for q in range(o // 8)]
            else:
                chains = [(0, 0, wt, 0, n16, 0), (0, 64, ws, 0, n16, n16), (1, 0, w2r, 0, n16, 2 * n16)]
                piece_col = [n16 * k + 8 * q for k in range(3) for q in range(o // 8)]
            piece_col += [-1] * (16 - len(piece_col))
            agg_w = torch.zeros(64, 128, device=w0.device)
            hid_b = torch.zeros(128, device=w0.device)
            for k, bk in enumerate((bt, bs, b2)):
                agg_w[:cout, k * o:k * o + half] = wg[:, k * half:(k + 1) * half]
                hid_b[k * o:k * o + half] = bk
            P["tail"] = dense.pack_block_tail(chains, agg_w, flat(wj)[:, :cs] if self.projection is not None else None,
                                              piece_col)
            P["tail_hid_bias"] = hid_b
            if nc:           # path 2 reads the spatially constant channels too: they shift its hidden bias per image
                wc = torch.zeros(128, nc, device=w0.device)
                wc[2 * o:2 * o + half] = flat(w2)[:, cs:]
                P["tail_hid_c"] = wc
        return P

    def forward_hl(self, x: dense.HL, const: Optional[torch.Tensor] = None,
                   sums: Optional[torch.Tensor] = None, out_sums: Optional[torch.Tensor] = None) -> dense.HL:
        """x: HL (B,T,H,W,.) holding the spatial input channels; const: (B*T, n_const) fp32 values of the spatially
        constant trailing channels (requires self.n_const == const.shape[1]); sums: optional precomputed per-image
        spatial sums of x (B*T, >= spatial channels), e.g. emitted by the lift-splat finalize kernel; out_sums (B*T, 64):
        receives the spatial sums of the block's output from the aggregation conv's epilogue (64-channel blocks)."""
        self._require_eval()
        nc = 0 if const is None else const.shape[1]
        assert nc == self.n_const, "set TemporalBlock.n_const to the number of spatially constant input channels"
        P = self.packed()
        B, T, H, W, _ = x.hi.shape
        dev = x.hi.device
        cin, half, cout, o, cs = self.in_channels, self.half_channels, self.out_channels, P["o"], P["cs"]
        n_img = B * T

        def const_bias(wc, pc):                    # per-image bias = conv bias + W[:, constant channels] . const
            if not nc:
                return None
            b = torch.empty((n_img, pc.bn), dtype=torch.float32, device=dev)
            dense.small_linear(const, wc, b, False, bias=pc.bias)
            return b

        if "tail" in P:
            return self._forward_fused(x, const, sums, out_sums, P, const_bias)
        m1 = P["m1"]
        ap = P["ap"]
        agg = dense.HL.empty(B, T, H, W, 3 * o, dev, cp=ap)
        # the last path also fills the padding channels of the concat tensor: its own padded output columns are exact
        # zeros (zero weights and bias), so storing up to 64 of them saves a separate fill
        tail = min(P["a2"].bn, ap - 2 * o)
        if 2 * o + tail < ap:                                    # fill what path 2's padded columns cannot reach
            agg.hi[..., 2 * o + tail:].zero_(); agg.lo[..., 2 * o + tail:].zero_()
        res = None
        if "a12" in P:         # [mid | path 2] in one launch
            mid = dense.HL.empty(B, T, H, W, 64, dev, cp=64)
            dense.conv(x, P["a12"], out=mid, n_store=64, relu=True, out2=agg, out2_coff=2 * o, n_store2=tail, relu2=True,
                       img_bias=const_bias(P.get("a12_c"), P["a12"]))
        else:
            mid = dense.conv(x, P["a1"], relu=True, img_bias=const_bias(P.get("a1_c"), P["a1"]))
            if "a2p" in P:     # [path 2 | projection] in one launch
                res = dense.HL.empty(B, T, H, W, cout, dev, cp=64)
                dense.conv(x, P["a2p"], out=agg, out_coff=2 * o, n_store=tail, relu=True, out2=res, out2_coff=0,
                           n_store2=64, relu2=False, img_bias=const_bias(P.get("a2p_c"), P["a2p"]))
            else:
                dense.conv(x, P["a2"], out=agg, out_coff=2 * o, n_store=tail, relu=True,
                           img_bias=const_bias(P.get("a2_c"), P["a2"]))
        if "bc" in P:          # one block-diagonal launch for both mid paths (they share a 64-channel block)
            dense.conv(mid, P["bc"], cin_off=0, out=agg, out_coff=0, n_store=2 * o, relu=True)
        else:
            dense.conv(mid, P["b"], cin_off=0, out=agg, out_coff=0, n_store=o, relu=True)
            dense.conv(mid, P["c"], cin_off=(m1 // 64) * 64, out=agg, out_coff=o, n_store=o, relu=True)
        pbias = None
        if self.use_pyramid_pooling:
            ph, pw = self.pyramid_pooling.pool_sizes[0][1:]
            assert (ph, pw) == (H, W), "pyramid pooling must span the whole map (as configured by TemporalModel)"
            if sums is None:
                sums = dense.spatial_sum(x)
            pbias = torch.empty((n_img, P["agg"].bn), dtype=torch.float32, device=dev)
            dense.pool_bias(sums, T, cin, H * W, True, P["pool_w1"], P["pool_b1"], P["pool_w2"], pbias, False,
                            const=const if nc else None, bias=P["agg"].bias)
        if res is None:
            if self.projection is not None:
                res = dense.conv(x, P["proj"], img_bias=const_bias(P.get("proj_c"), P["proj"]))
            else:
                assert nc == 0, "an identity skip cannot carry spatially constant extra channels"
                res = x
        return dense.conv(agg, P["agg"], relu=True, img_bias=pbias, residual=res, res_after_act=True, col_sums=out_sums)

    def _forward_fused(self, x, const, sums, out_sums, P, const_bias):
        """Entry convolutions of paths 0 / 1 as one launch, then the whole tail of the block (both spatio-temporal
        convolutions, path 2, aggregation, pyramid-pooling bias, projection / identity residual, output column sums) in
        the back-to-back kernel: the concat tensor and the separate path-2 / projection passes over x disappear."""
        B, T, H, W, _ = x.hi.shape
        dev = x.hi.device
        n_img = B * T
        nc = 0 if const is None else const.shape[1]
        mid = dense.conv(x, P["a1"], relu=True, img_bias=const_bias(P.get("a1_c"), P["a1"]))
        if nc:
            hid = torch.empty((n_img, 128), dtype=torch.float32, device=dev)
            dense.small_linear(const, P["tail_hid_c"], hid, False, bias=P["tail_hid_bias"])
        else:
            key = ("tail_hid", n_img)
            if key not in P:
                P[key] = P["tail_hid_bias"].unsqueeze(0).expand(n_img, -1).contiguous()
            hid = P[key]
        if self.use_pyramid_pooling:
            ph, pw = self.pyramid_pooling.pool_sizes[0][1:]
            assert (ph, pw) == (H, W), "pyramid pooling must span the whole map (as configured by TemporalModel)"
            if sums is None:
                sums = dense.spatial_sum(x)
            pbias = torch.empty((n_img, 64), dtype=torch.float32, device=dev)
            dense.pool_bias(sums, T, self.in_channels, H * W, True, P["pool_w1"], P["pool_b1"], P["pool_w2"], pbias, False,
                            const=const if nc else None, bias=P["agg"].bias)
        else:
            key = ("tail_agg_bias", n_img)
            if key not in P:
                P[key] = P["agg"].bias.unsqueeze(0).expand(n_img, -1).contiguous()
            pbias = P[key]
        rbias = None
        if self.projection is not None:
            if nc:
                rbias = torch.empty((n_img, 64), dtype=torch.float32, device=dev)
                dense.small_linear(const, P["proj_c"], rbias, False, bias=P["proj"].bias)
            else:
                key = ("tail_res_bias", n_img)
                if key not in P:
                    P[key] = P["proj"].bias.unsqueeze(0).expand(n_img, -1).contiguous()
                rbias = P[key]
        y = dense.block_tail(mid, x, P["tail"], hid, pbias, rbias, col_sums=out_sums)
        y.c = self.out_channels
        return y

    def forward(self, *inputs):
        """x (B, C, T, H, W) fp32 -> (B, Cout, T, H, W) fp32, like the reference module."""
        (x,) = inputs
        assert self.n_const == 0
        y = self.forward_hl(dense.from_f32(x.permute(0, 2, 1, 3, 4)))
        return dense.to_f32(y, 0, self.out_channels).permute(0, 2, 1, 3, 4)
