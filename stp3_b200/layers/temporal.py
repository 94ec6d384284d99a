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

SpatialGRU and Dual_GRU (bottom of the file) are the eval-only conv-GRUs of the prediction stage (DESIGN.md §3.16).

Train mode (batch statistics, autograd) runs only inside TemporalModel, which wraps the whole block stack in one
autograd node (temporal_model._TemporalBlocksTrainFn) built on _train_forward / _train_backward below; a block called
on its own keeps refusing train().
"""
import os
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn

from .. import dense, dense_train
from ._packing import PackedModule
from .convolutions import Bottleblock, PredictModule


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

    def _require_eval(self):
        if self.training:
            raise NotImplementedError(
                "TemporalBlock: train mode runs through TemporalModel, which trains its blocks and its head together "
                "(TemporalModel.train()); a block on its own implements the inference forward only -- call .eval()")

    # ------------------------------------------------------------------------------------------------ train mode
    def _x_convs(self):
        """The 1x1x1 convolutions that read x, in the row order of the backward's pre-BN gradient tensor: the three
        entry convolutions of the paths, then the projection."""
        p0, p1, p2 = self.convolution_paths
        convs = [p0[0].conv, p1[0].conv, p2.conv]
        return convs + ([self.projection[0]] if self.projection is not None else [])

    def _train_forward(self, x: torch.Tensor, const: Optional[torch.Tensor], B: int, T: int):
        """x (B*T, H, W, cs) fp32 channels-last: the spatial input channels; const (B*T, n_const) fp32 or None: the
        spatially constant ones.  Every BatchNorm3d uses batch statistics over B*T*H*W (the pooled branch's over the B*T
        values) and updates its running statistics.  -> (y (B*T, H, W, cout) fp32, tape for _train_backward)."""
        N, H, W, cs = x.shape
        nc = 0 if const is None else const.shape[1]
        assert nc == self.n_const and cs + nc == self.in_channels
        if self.projection is None and nc:
            raise NotImplementedError("TemporalBlock: an identity skip cannot carry spatially constant extra channels")
        h, cout = self.half_channels, self.out_channels
        dev = x.device
        TT = dense_train
        mode = TT.amp_mode()
        x_hl = TT.to_hl(x, **TT.amp_kw(mode))

        def x_conv(conv):                  # 1x1x1 convolution of x; the constant channels enter as a per-image bias
            w = conv.weight.detach().float().reshape(conv.out_channels, -1)
            ib = None
            if nc:
                ib = torch.zeros((N, dense.out_tile(w.shape[0])), dtype=torch.float32, device=dev)
                dense.small_linear(const, w[:, cs:].contiguous(), ib, False)
            return TT.conv_raw(x_hl, w[:, :cs].reshape(w.shape[0], cs, 1, 1).contiguous(), 1, img_bias=ib)

        # the three paths write their activated outputs side by side: the aggregation's spatial input
        cat = torch.empty((N, H, W, 3 * h), dtype=torch.float32, device=dev)
        entry, mids = [], []
        for i, path in enumerate(self.convolution_paths):
            e = path[0] if i < 2 else path
            raw = x_conv(e.conv)
            st = TT.bn_stats_module(raw, e.norm)
            if i < 2:
                y, y_hl = TT.bn_apply(raw, st, e.norm.weight, e.norm.bias, relu=True, **TT.amp_kw(mode))
                cc = path[1]
                y_hl = dense.HL(y_hl.hi.view(B, T, *y_hl.hi.shape[2:]),
                                y_hl.lo.view(B, T, *y_hl.lo.shape[2:]) if y_hl.lo is not None else None, h)
                raw2 = TT.conv_raw(y_hl, cc.conv.weight, 1)
                st2 = TT.bn_stats_module(raw2, cc.norm)
                TT.bn_apply(raw2, st2, cc.norm.weight, cc.norm.bias, relu=True, hl=False, y_out=cat[..., i * h:(i + 1) * h])
                mids.append((cc, raw2, st2))
            else:
                y = cat[..., 2 * h:]
                TT.bn_apply(raw, st, e.norm.weight, e.norm.bias, relu=True, hl=False, y_out=y)
            entry.append((e, raw, st, y))
        agg = self.aggregation[0]
        wg = agg.conv.weight.detach().float().reshape(cout, -1)
        # x: what the 1x1x1 convolutions' weight gradient reads (under autocast the plane they multiplied, not the fp32
        # block input)
        tape = {"x": x if mode is None else x_hl, "shape": (N, H, W, cs), "const": const, "B": B, "T": T, "cat": cat,
                "entry": entry, "mids": mids, "mode": mode}
        pbias = None
        if self.use_pyramid_pooling:
            # per-frame means -> temporal pair mean (AvgPool3d with count_include_pad=False: T + 1 frames) -> 1x1x1 ->
            # BatchNorm over the B*(T+1) values -> ReLU -> last frame dropped (that order is the reference's,
            # temporal.py:414): spatially constant, so it enters the aggregation as a per-image bias and the broadcast
            # map is never built
            ph, pw = self.pyramid_pooling.pool_sizes[0][1:]
            assert (ph, pw) == (H, W), "pyramid pooling must span the whole map (as configured by TemporalModel)"
            pcbr = self.pyramid_pooling.features[0].conv_bn_relu
            red = pcbr.conv.out_channels
            mean = torch.empty((N, self.in_channels), dtype=torch.float32, device=dev)
            mean[:, :cs] = TT.image_channel_sums(x) * (1.0 / (H * W))
            if nc:
                mean[:, cs:] = const
            m = TT.temporal_pair_mean(mean, T)
            Np = m.shape[0]
            v_raw = torch.empty((Np, 1, 1, red), dtype=torch.float32, device=dev)
            dense.small_linear(m, pcbr.conv.weight.detach().float().reshape(red, -1).contiguous(), v_raw.view(Np, red),
                               False)
            pst = TT.bn_stats_module(v_raw, pcbr.norm)
            v_full, _ = TT.bn_apply(v_raw, pst, pcbr.norm.weight, pcbr.norm.bias, relu=True, hl=False)
            v = v_full.view(B, T + 1, red)[:, :T].reshape(N, 1, 1, red).contiguous()
            pbias = torch.zeros((N, dense.out_tile(cout)), dtype=torch.float32, device=dev)
            dense.small_linear(v.view(N, red), wg[:, 3 * h:].contiguous(), pbias, False)
            tape.update(m=m, v_raw=v_raw, pst=pst, v_full=v_full, v=v)
        araw = TT.conv_raw(TT.to_hl(cat, **TT.amp_kw(mode)), wg[:, :3 * h].reshape(cout, 3 * h, 1, 1).contiguous(), 1, img_bias=pbias)
        ast = TT.bn_stats_module(araw, agg.norm)
        ya, _ = TT.bn_apply(araw, ast, agg.norm.weight, agg.norm.bias, relu=True, hl=False)
        tape.update(araw=araw, ast=ast, ya=ya)
        if self.projection is not None:
            jbn = self.projection[1]
            jraw = x_conv(self.projection[0])
            jst = TT.bn_stats_module(jraw, jbn)
            out, _ = TT.bn_apply(jraw, jst, jbn.weight, jbn.bias, relu=False, hl=False)
            out.add_(ya)
            tape.update(jraw=jraw, jst=jst)
        else:
            out = ya + x
        return out, tape

    def _train_backward(self, tape, g: torch.Tensor, need_x: bool):
        """Reverse walk of _train_forward: g = dL/dy (B*T, H, W, cout) contiguous fp32 -> (dL/dx (B*T, H, W, cs) or
        None, {parameter: gradient}).  No gradient reaches the constant channels (host-derived input data)."""
        TT = dense_train
        x, const, B, T, cat = tape["x"], tape["const"], tape["B"], tape["T"], tape["cat"]
        mode = tape["mode"]       # the spatial convolutions' precision; the pooling branch's products stay fp32
        op = lambda t: TT.operand(t, mode)     # noqa: E731  (one plane per gradient under autocast)
        N, H, W, cs = tape["shape"]
        nc = 0 if const is None else const.shape[1]
        h, cout = self.half_channels, self.out_channels
        dev = cat.device
        grads = {}
        convs = self._x_convs()
        K = 3 * h + (cout if self.projection is not None else 0)
        # pre-BN gradients of every 1x1x1 convolution that reads x, side by side: one wgrad and one transposed
        # convolution serve all of them
        graw = torch.empty((N, H, W, K), dtype=torch.float32, device=dev)
        if self.projection is not None:
            jbn = self.projection[1]
            _, grads[jbn.weight], grads[jbn.bias], _ = TT.bn_backward(g, tape["jraw"], tape["jst"], jbn.weight, None,
                                                                      dx_out=graw[..., 3 * h:])
        agg = self.aggregation[0]
        wg = agg.conv.weight.detach().float().reshape(cout, -1)
        ga, grads[agg.norm.weight], grads[agg.norm.bias], _ = TT.bn_backward(g, tape["araw"], tape["ast"],
                                                                            agg.norm.weight, tape["ya"])
        ga_op = op(ga)
        dw_agg = TT.conv_wgrad(cat, ga_op, 1, 1, 1, **TT.amp_kw(mode)).reshape(cout, 3 * h)
        g_cat = TT.conv_dgrad(ga_op, wg[:, :3 * h].reshape(cout, 3 * h, 1, 1), 1, H, W, **TT.amp_kw(mode))
        gx_pool = None
        if self.use_pyramid_pooling:
            pcbr = self.pyramid_pooling.features[0].conv_bn_relu
            red = pcbr.conv.out_channels
            gsum = TT.image_channel_sums(ga)
            v = tape["v"]
            dw_agg = torch.cat([dw_agg, TT.conv_wgrad(v, gsum.view(N, 1, 1, cout), 1, 1, 1).reshape(cout, red)], 1)
            g_vk = torch.empty((N, red), dtype=torch.float32, device=dev)
            dense.small_linear(gsum, wg[:, 3 * h:].t().contiguous(), g_vk, False)
            m = tape["m"]
            Np = m.shape[0]
            g_v = torch.zeros((B, T + 1, red), dtype=torch.float32, device=dev)    # the dropped frame gets none
            g_v[:, :T] = g_vk.view(B, T, red)
            g_v, grads[pcbr.norm.weight], grads[pcbr.norm.bias], _ = TT.bn_backward(
                g_v.view(Np, 1, 1, red), tape["v_raw"], tape["pst"], pcbr.norm.weight, tape["v_full"])
            grads[pcbr.conv.weight] = TT.conv_wgrad(m.view(Np, 1, 1, -1), g_v, 1, 1, 1).view_as(pcbr.conv.weight)
            if need_x:
                # d mean = pair-mean adjoint of W1^T g_v; its spatial channels spread evenly over the H*W pixels and
                # enter the input gradient as the per-image bias of the transposed convolution below
                wp = pcbr.conv.weight.detach().float().reshape(red, -1)
                g_m = torch.empty((Np, self.in_channels), dtype=torch.float32, device=dev)
                dense.small_linear(g_v.view(Np, red), wp.t().contiguous(), g_m, False)
                g_mean = TT.temporal_pair_mean(g_m, T, adjoint=True)
                gx_pool = torch.zeros((N, dense.out_tile(cs)), dtype=torch.float32, device=dev)
                gx_pool[:, :cs] = g_mean[:, :cs] * (1.0 / (H * W))
        grads[agg.conv.weight] = dw_agg.view_as(agg.conv.weight)
        for i, (e, raw, st, y) in enumerate(tape["entry"]):
            sl = slice(i * h, (i + 1) * h)
            gi = g_cat[..., sl]
            if i < 2:
                cc, raw2, st2 = tape["mids"][i]
                g2, grads[cc.norm.weight], grads[cc.norm.bias], _ = TT.bn_backward(gi, raw2, st2, cc.norm.weight,
                                                                                  cat[..., sl])
                kt = cc.conv.kernel_size[0]
                g2_op = op(g2) if mode is not None else g2.view(B, T, H, W, h)
                grads[cc.conv.weight] = TT.conv_wgrad(y.view(B, T, H, W, h), g2_op, 3, 3, 1, kt=kt, **TT.amp_kw(mode))
                gi = TT.conv_dgrad(g2 if mode is None else g2_op, cc.conv.weight, 1, H, W, T=T, **TT.amp_kw(mode))
            _, grads[e.norm.weight], grads[e.norm.bias], _ = TT.bn_backward(gi, raw, st, e.norm.weight, y,
                                                                            dx_out=graw[..., sl])
        graw_op = op(graw)
        dw_x = TT.conv_wgrad(x, graw_op, 1, 1, 1, **TT.amp_kw(mode)).reshape(K, cs)
        if nc:
            # the constant channels' columns: sum over images of (per-image sums of the pre-BN gradient) x const
            gs = TT.image_channel_sums(graw)
            dw_x = torch.cat([dw_x, TT.conv_wgrad(const.view(N, 1, 1, nc), gs.view(N, 1, 1, K), 1, 1, 1).reshape(K, nc)], 1)
        row = 0
        for conv in convs:
            grads[conv.weight] = dw_x[row:row + conv.out_channels].reshape(conv.weight.shape).contiguous()
            row += conv.out_channels
        gx = None
        if need_x:
            w_x = torch.cat([conv.weight.detach().float().reshape(conv.out_channels, -1)[:, :cs] for conv in convs], 0)
            gx = TT.conv_dgrad(graw_op, w_x.reshape(K, cs, 1, 1).contiguous(), 1, H, W, img_bias=gx_pool,
                               **TT.amp_kw(mode))
            if self.projection is None:
                gx.add_(g)
        return gx, grads

    def forward(self, *inputs):
        """x (B, C, T, H, W) fp32 -> (B, Cout, T, H, W) fp32, like the reference module."""
        (x,) = inputs
        assert self.n_const == 0
        y = self.forward_hl(dense.from_f32(x.permute(0, 2, 1, 3, 4)))
        return dense.to_f32(y, 0, self.out_channels).permute(0, 2, 1, 3, 4)


# ------------------------------------------------------------------------------------------------ prediction stage
def _gru_pack(conv_update, conv_reset, conv_tilde, input_size, hidden_size):
    """The two convolutions of a conv-GRU cell over one buffer [h | x | (1 - r) * h] (64-channel slots; x at 64): the
    update and reset gates as one 128-column convolution of channels [0, 128), the proposal as a convolution of
    channels [64, 192).  The reference concatenates (x, h) in that order; in_layout maps its input channels."""
    g_w = torch.cat([conv_update.weight, conv_reset.weight]).detach().float()
    g_b = torch.cat([conv_update.bias, conv_reset.bias]).detach().float()
    gate = dense.pack_conv(g_w, g_b, in_layout=[(0, input_size, 64), (input_size, hidden_size, 0)], cin_p=128)
    prop = dense.pack_conv(conv_tilde.weight.detach().float(), conv_tilde.bias.detach().float(),
                           in_layout=[(0, input_size, 0), (input_size, hidden_size, 64)], cin_p=128)
    return gate, prop


def _gru_step(buf: dense.HL, gate: dense.PackedConv, prop: dense.PackedConv, out2=None):
    """One conv-GRU cell on buf = [h | x | scratch]: buf's h slot becomes (1 - u) * h + u * h_tilde (and out2 too).
    The gates leave the convolution raw and the two per-pixel kernels apply the sigmoids: stp3_conv_fwd's sigmoid
    exists only for its NCHW fp32 output (the instance-center head; the channels-last fp32 output refuses it and the
    hi/lo output has none), and the kernels that consume the gates read channels-last hi/lo."""
    g = dense.conv(buf, gate)                                   # raw [update | reset] gates, (B, 1, H, W, 128)
    dense.gru_gates((g, 64), buf, (buf, 128), 64)
    h_tilde = dense.conv(buf, prop, cin_off=64)
    dense.gru_update(g, buf, h_tilde, buf, 64, out2=out2)


class _PredictGRU(PredictModule):
    @staticmethod
    def _check_sizes(input_size, hidden_size):
        if hidden_size != 64 or input_size > 64:
            raise NotImplementedError(f"conv-GRU with input {input_size} / hidden {hidden_size}: the sm_90a cell keeps "
                                      "64-channel slots (the reference's configs use hidden 64, inputs 32 and 64)")


class SpatialGRU(_PredictGRU):
    """Convolutional GRU over a sequence (temporal.py:11-58), eval only: gates sigmoid(conv3x3([x, h])), proposal
    conv3x3([x, (1 - r) * h]), h = (1 - u) * h + u * h_tilde, and a 1x1 conv_decoder (no bias) on every state."""

    def __init__(self, input_size, hidden_size, gru_bias_init=0.0):
        super().__init__()
        if gru_bias_init != 0.0:
            raise NotImplementedError("SpatialGRU: gru_bias_init != 0 is not used by the reference")
        self._check_sizes(input_size, hidden_size)
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.gru_bias_init = gru_bias_init
        self.conv_update = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_reset = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_state_tilde = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_decoder = nn.Conv2d(hidden_size, input_size, kernel_size=1, bias=False)

    def _pack(self):
        gate, prop = _gru_pack(self.conv_update, self.conv_reset, self.conv_state_tilde, self.input_size,
                               self.hidden_size)
        w = self.conv_decoder.weight.detach().float()
        return {"gate": gate, "prop": prop, "dec": dense.pack_conv(w, torch.zeros(w.shape[0], device=w.device))}

    def forward_hl(self, frames, state) -> dense.HL:
        """frames: the input sequence as a list of (HL, frame index) -- frame t of every sample is x_t; state:
        (HL, frame index) of the initial hidden state.  Returns HL (B, len(frames), H, W, 64): conv_decoder of every
        state."""
        self._require_eval()
        P = self.packed()
        x0 = frames[0][0]
        B, _, H, W, _ = x0.hi.shape
        dev = x0.hi.device
        n = len(frames)
        buf = dense.HL.zeros(B, 1, H, W, 192, dev, cp=192)         # [h | x | (1 - r) * h]
        states = dense.HL.empty(B, n, H, W, 64, dev, cp=64)
        dense.hl_copy((state[0], 0, state[1]), buf, 64, T=1)
        for t, (src, f) in enumerate(frames):
            dense.hl_copy((src, 0, f), (buf, 64), self.input_size + (-self.input_size) % 8, T=1)
            _gru_step(buf, P["gate"], P["prop"], out2=(states, 0, t))
        return dense.conv(states, P["dec"])

    def forward(self, x, state=None):
        """x (B, T, C, H, W) fp32, state (B, hidden, H, W) fp32 (zeros when None) -> (B, T, input_size, H, W) fp32."""
        B, T = x.shape[:2]
        xs = dense.from_f32(x)
        h = dense.from_f32((state if state is not None else x.new_zeros(B, self.hidden_size, *x.shape[3:])).unsqueeze(1))
        y = self.forward_hl([(xs, t) for t in range(T)], (h, 0))
        return dense.to_f32(y, 0, self.input_size)


class Dual_GRU(_PredictGRU):
    """The future recurrence of FuturePrediction (temporal.py:60-160), eval only with mixture=True.  gru_cell_2 warms up
    over the present states; each future step runs gru_cell_1 (input: the latent sample) and gru_cell_2 ->
    conv_decoder_2, and the trusting gate mixes the two states: p = softmax(conv1x1(Bottleblock([s1, s2]))),
    mix = s2 * p0 + s1 * p1, which becomes both recurrences' state and the step's output."""

    def __init__(self, in_channels, latent_dim, n_future, mixture=True, gru_bias_init=0.0):
        super().__init__()
        if gru_bias_init != 0.0:
            raise NotImplementedError("Dual_GRU: gru_bias_init != 0 is not used by the reference")
        input_size = in_channels
        hidden_size = latent_dim
        self._check_sizes(input_size, hidden_size)
        self.n_future = n_future
        self.mixture = mixture
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.gru_bias_init = gru_bias_init
        self.conv_update_1 = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_reset_1 = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_state_tilde_1 = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_update_2 = nn.Conv2d(hidden_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_reset_2 = nn.Conv2d(hidden_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_state_tilde_2 = nn.Conv2d(hidden_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_decoder_2 = nn.Conv2d(hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.trusting_gate = nn.Sequential(
            Bottleblock(hidden_size + hidden_size, hidden_size),
            nn.Conv2d(hidden_size, 2, kernel_size=1, bias=False)
        )

    def _pack(self):
        P = {}
        P["gate1"], P["prop1"] = _gru_pack(self.conv_update_1, self.conv_reset_1, self.conv_state_tilde_1,
                                           self.input_size, self.hidden_size)
        P["gate2"], P["prop2"] = _gru_pack(self.conv_update_2, self.conv_reset_2, self.conv_state_tilde_2,
                                           self.hidden_size, self.hidden_size)
        P["dec2"] = dense.pack_conv(self.conv_decoder_2.weight.detach().float(),
                                    self.conv_decoder_2.bias.detach().float())
        P["trust_w"] = self.trusting_gate[1].weight.detach().float().reshape(2, self.hidden_size).contiguous()
        return P

    def forward_hl(self, x: Optional[dense.HL], state: dense.HL, out: dense.HL, out_t0: int = 0):
        """x: HL (B, 1, H, W, >= input_size) the latent sample, or None for zeros; state: HL (B, S, H, W, 64) the
        present states.  The n_future predicted states go to frames [out_t0, out_t0 + n_future) of out."""
        self._require_eval()
        if not self.mixture:
            raise NotImplementedError("Dual_GRU: mixture=False is not built (every reference config mixes)")
        P = self.packed()
        B, S, H, W, _ = state.hi.shape
        dev = state.hi.device
        a1 = dense.HL.zeros(B, 1, H, W, 192, dev, cp=192)      # cell 1: [s1 | x | (1 - r) * s1]
        a2 = dense.HL.zeros(B, 1, H, W, 192, dev, cp=192)      # cell 2: [h | s2 | (1 - r) * h]
        mix = dense.HL.empty(B, 1, H, W, 128, dev, cp=128)     # [s1 | s2], the trusting gate's input
        if x is not None:
            dense.hl_copy(x, (a1, 64), self.input_size, T=1)
        dense.hl_copy((state, 0, 0), a2, 64, T=1)
        for t in range(S - 1):                                   # warm-up of gru_cell_2 over the present states
            dense.hl_copy((state, 0, t), (a2, 64), 64, T=1)
            _gru_step(a2, P["gate2"], P["prop2"])
        dense.hl_copy((state, 0, S - 1), a1, 64, T=1)
        dense.hl_copy((state, 0, S - 1), (a2, 64), 64, T=1)
        gate_blk = self.trusting_gate[0]
        for t in range(self.n_future):
            _gru_step(a1, P["gate1"], P["prop1"], out2=(mix, 0))     # s1 -> a1[0:64] and mix[0:64]
            _gru_step(a2, P["gate2"], P["prop2"])
            dense.conv(a2, P["dec2"], out=mix, out_coff=64)          # s2 = conv_decoder_2(h) -> mix[64:128]
            g = gate_blk.forward_hl(mix)
            dense.trust_mix(g, P["trust_w"], (mix, 0), (mix, 64), [(a1, 0), (a2, 64), (out, 0, out_t0 + t)], 64, T=1)
        return out

    def forward(self, x, state):
        """x (B, 1, input_size, H, W) fp32, state (B, S, hidden, H, W) fp32 -> (B, n_future, hidden, H, W) fp32."""
        B, S, _, H, W = state.shape
        out = dense.HL.empty(B, self.n_future, H, W, 64, state.device, cp=64)
        self.forward_hl(dense.from_f32(x), dense.from_f32(state), out)
        return dense.to_f32(out, 0, self.hidden_size)
