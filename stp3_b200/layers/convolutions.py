"""2-D building blocks of the BEV path with the reference's constructor signatures and parameter names
(stp3/layers/convolutions.py:183-280) so checkpoints load unchanged; forward() runs on the wgmma kernels.

  UpsamplingAdd  : bilinear x2 -> 1x1 conv -> BN, + skip.   Executed as 1x1 conv + folded BN at LOW resolution and a
                   fused upsample+add kernel (the interpolation weights sum to one, so the affine map commutes).
  ASPP / DeepLabHead : the five ASPP branches write straight into one channels-last concat tensor; the global-pool
                   branch is spatially constant and becomes a per-image bias of the 1x1 projection.
"""
import os
from typing import Optional

import torch
import torch.nn as nn

from .. import dense
from ._packing import PackedModule


class UpsamplingAdd(PackedModule):
    def __init__(self, in_channels, out_channels, scale_factor=2):
        super().__init__()
        assert scale_factor == 2, "the fused kernel implements the reference's only use: scale_factor=2"
        self.upsample_layer = nn.Sequential(
            nn.Upsample(scale_factor=scale_factor, mode='bilinear', align_corners=False),
            nn.Conv2d(in_channels, out_channels, kernel_size=1, padding=0, bias=False),
            nn.BatchNorm2d(out_channels),
        )

    def _pack(self):
        w, b = dense.fold_bn(self.upsample_layer[1].weight, self.upsample_layer[2])
        return dense.pack_conv(w, b)

    def forward_hl(self, x: dense.HL, skip: dense.HL, skip_coff: int = 0) -> dense.HL:
        self._require_eval()
        pc = self.packed()
        low = dense.conv(x, pc)                                   # 1x1 + BN at low resolution
        return dense.upsample2x_add(low, skip, pc.bn if pc.cout % 8 else pc.cout, skip_coff)

    def forward(self, x, x_skip):
        """x (N,Cin,h,w), x_skip (N,Cout,2h,2w) fp32 -> (N,Cout,2h,2w), like the reference module."""
        y = self.forward_hl(dense.from_f32(x.unsqueeze(1)), dense.from_f32(x_skip.unsqueeze(1)))
        return dense.to_f32(y, 0, x_skip.shape[1]).squeeze(1)


class ASPPConv(nn.Sequential):
    def __init__(self, in_channels, out_channels, dilation):
        super().__init__(nn.Conv2d(in_channels, out_channels, 3, padding=dilation, dilation=dilation, bias=False),
                         nn.BatchNorm2d(out_channels), nn.ReLU())


class ASPPPooling(nn.Sequential):
    def __init__(self, in_channels, out_channels):
        super().__init__(nn.AdaptiveAvgPool2d(1), nn.Conv2d(in_channels, out_channels, 1, bias=False),
                         nn.BatchNorm2d(out_channels), nn.ReLU())


class ASPP(nn.Module):
    def __init__(self, in_channels, atrous_rates, out_channels=256):
        super().__init__()
        branches = [nn.Sequential(nn.Conv2d(in_channels, out_channels, 1, bias=False), nn.BatchNorm2d(out_channels),
                                  nn.ReLU())]
        branches += [ASPPConv(in_channels, out_channels, r) for r in tuple(atrous_rates)]
        branches.append(ASPPPooling(in_channels, out_channels))
        self.convs = nn.ModuleList(branches)
        self.project = nn.Sequential(nn.Conv2d(len(self.convs) * out_channels, out_channels, 1, bias=False),
                                     nn.BatchNorm2d(out_channels), nn.ReLU(), nn.Dropout(0.5))
        self.rates = tuple(atrous_rates)


class DeepLabHead(nn.Sequential, PackedModule):
    """ASPP(12,24,36) -> 3x3 conv/BN/ReLU -> 1x1 conv(+bias)  (convolutions.py:272-280)."""

    def __init__(self, in_channels, num_classes, hidden_channel=256):
        nn.Sequential.__init__(
            self,
            ASPP(in_channels, [12, 24, 36], hidden_channel),
            nn.Conv2d(hidden_channel, hidden_channel, 3, padding=1, bias=False),
            nn.BatchNorm2d(hidden_channel),
            nn.ReLU(),
            nn.Conv2d(hidden_channel, num_classes, 1),
        )
        self.hidden = hidden_channel
        self.in_channels = in_channels
        self.num_classes = num_classes

    def _pack(self, extent=None):
        aspp: ASPP = self[0]
        h = self.hidden
        assert h % 64 == 0, "hidden channels must be a multiple of 64 (128 in the temporal model, 64 in the encoder)"
        P = {}
        w, b = dense.fold_bn(aspp.convs[0][0].weight, aspp.convs[0][1])
        P["b0"] = dense.pack_conv(w, b, bn=h)
        for i, r in enumerate(aspp.rates):
            w, b = dense.fold_bn(aspp.convs[1 + i][0].weight, aspp.convs[1 + i][1])
            P[f"b{i + 1}"] = dense.pack_conv(w, b, dilation=r, bn=h)
        nb = 1 + len(aspp.rates)
        wp, bp = dense.fold_bn(aspp.convs[nb][1].weight, aspp.convs[nb][2])           # pooling branch 1x1 + BN
        P["pool_w1"], P["pool_b1"] = wp.reshape(h, -1).contiguous(), bp.contiguous()
        wproj, bproj = dense.fold_bn(aspp.project[0].weight, aspp.project[1])         # (h, (nb+1)*h, 1, 1)
        P["proj"] = dense.pack_conv(wproj[:, :nb * h].contiguous(), bproj, bn=h)
        P["pool_w2"] = wproj[:, nb * h:(nb + 1) * h].reshape(h, h).contiguous()
        w, b = dense.fold_bn(self[1].weight, self[2])
        P["conv3"] = dense.pack_conv(w, b, bn=h)
        P["cls"] = dense.pack_conv(self[4].weight.detach().float(), self[4].bias.detach().float())
        P["nb"] = nb
        # hidden = 128, dilations that fit signed-byte taps: branches + projection as one back-to-back kernel
        if h == 128 and nb <= 4 and max(aspp.rates) <= 127 and os.environ.get("STP3_ASPP_FUSED", "1") != "0":
            br = []
            w, b = dense.fold_bn(aspp.convs[0][0].weight, aspp.convs[0][1])
            br.append((w, b, 1))
            for i, r in enumerate(aspp.rates):
                w, b = dense.fold_bn(aspp.convs[1 + i][0].weight, aspp.convs[1 + i][1])
                br.append((w, b, r))
            P["fused"] = dense.pack_aspp(br, wproj[:, :nb * h].reshape(h, nb * h), bproj)
            if self.num_classes <= 64:
                # the tail 3x3 conv/BN/ReLU -> 1x1 classifier through the same back-to-back kernel (one branch): the
                # 128-channel intermediate stays on chip
                w3, b3 = dense.fold_bn(self[1].weight, self[2])
                P["tail"] = dense.pack_aspp([(w3, b3, 1)], self[4].weight.detach().float().reshape(self.num_classes, h),
                                            self[4].bias.detach().float())
        return P

    def forward_hl(self, x: dense.HL, out: Optional[dense.HL] = None, sums: Optional[torch.Tensor] = None) -> dense.HL:
        """x: HL (B,T,H,W,>=Cin) -> HL with num_classes channels (every (b,t) image independently); sums: optional
        (B*T, >= Cin) spatial sums of x when the producer already has them."""
        self._require_eval()
        P = self.packed()
        B, T, H, W, _ = x.hi.shape
        h, nb = self.hidden, P["nb"]
        dev = x.hi.device
        if sums is None:
            sums = dense.spatial_sum(x)
        pbias = torch.empty((B * T, P["proj"].bn), dtype=torch.float32, device=x.hi.device)
        dense.pool_bias(sums, T, self.in_channels, H * W, False, P["pool_w1"], P["pool_b1"], P["pool_w2"], pbias, False,
                        bias=P["proj"].bias)
        if "fused" in P and x.hi.shape[-1] == P["fused"].cin_p:
            y = dense.aspp_fused(x, P["fused"], pbias)                  # the concat tensor is never materialised
        else:
            cat = dense.HL.empty(B, T, H, W, nb * h, dev, cp=nb * h)
            for i in range(nb):
                dense.conv(x, P[f"b{i}"], out=cat, out_coff=i * h, relu=True)
            y = dense.conv(cat, P["proj"], relu=True, img_bias=pbias)   # Dropout(0.5) is the identity in eval mode
        if "tail" in P and out is None:
            key = ("tail_bias", B * T)
            if key not in P:                   # the classifier's bias as a (constant) per-image table, built once
                P[key] = P["tail"].proj_bias.unsqueeze(0).expand(B * T, -1).contiguous()
            return dense.aspp_fused(y, P["tail"], P[key], relu=False, n_store=64, c_out=self.num_classes)
        y = dense.conv(y, P["conv3"], relu=True)
        return dense.conv(y, P["cls"], out=out)

    def forward(self, x):
        """x (N,Cin,H,W) fp32 -> (N,num_classes,H,W) fp32."""
        y = self.forward_hl(dense.from_f32(x.unsqueeze(1)))
        return dense.to_f32(y, 0, self.num_classes).squeeze(1)


class UpsamplingConcat(PackedModule):
    """bilinear x2 of the coarse map, concat behind the fine map, two 3x3 conv/BN/ReLU (convolutions.py:183-201).
    The upsample kernel writes straight into its channel window of the concat tensor."""

    def __init__(self, in_channels, out_channels, scale_factor=2):
        super().__init__()
        assert scale_factor == 2
        self.upsample = nn.Upsample(scale_factor=scale_factor, mode='bilinear', align_corners=False)
        self.conv = nn.Sequential(
            nn.Conv2d(in_channels, out_channels, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(out_channels),
            nn.ReLU(inplace=True),
            nn.Conv2d(out_channels, out_channels, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(out_channels),
            nn.ReLU(inplace=True),
        )
        self.in_channels, self.out_channels = in_channels, out_channels

    def _pack(self):
        w0, b0 = dense.fold_bn(self.conv[0].weight, self.conv[1])
        w1, b1 = dense.fold_bn(self.conv[3].weight, self.conv[4])
        return {"c0": (w0, b0), "c1": dense.pack_conv(w1, b1)}

    def forward_hl(self, coarse: dense.HL, fine_f32: torch.Tensor, out_f32: Optional[torch.Tensor] = None,
                   out_f32_nhwc: bool = False):
        """coarse: HL (B,1,h,w,.) with coarse.c real channels; fine_f32: (B, Cf, 2h, 2w) fp32.
        out_f32: optional fp32 destination written by the last convolution's epilogue instead of hi/lo planes --
        (B, Cout, 2h, 2w) like the reference, or channels-last (B, 2h, 2w, Cout) with out_f32_nhwc (the layout the
        lift-splat fetches as one TMA box per tile)."""
        self._require_eval()
        P = self.packed()
        cf, cc = fine_f32.shape[1], coarse.c
        assert cf + cc == self.in_channels and cf % 8 == 0 and cc % 8 == 0
        key = ("c0p", cf, cc)
        if key not in P:     # first conv packed for the physical layout [fine | coarse]
            P[key] = dense.pack_conv(P["c0"][0], P["c0"][1], in_layout=[(0, cf, 0), (cf, cc, cf)])
        cat = dense.from_f32(fine_f32.unsqueeze(1), cp=dense.pad_to(cf + cc))
        dense.upsample2x_add(coarse, None, cc, out=cat, out_coff=cf)
        y = dense.conv(cat, P[key], relu=True)
        if out_f32 is None:
            return dense.conv(y, P["c1"], relu=True)
        B = y.hi.shape[0]
        shape = (B, *y.hi.shape[2:4], self.out_channels) if out_f32_nhwc else (B, self.out_channels, *y.hi.shape[2:4])
        assert tuple(out_f32.shape) == shape and out_f32.dtype == torch.float32 and out_f32.is_contiguous()
        dense.conv(y, P["c1"], relu=True, out_f32=out_f32, n_valid=self.out_channels, out_f32_nhwc=out_f32_nhwc, store=False)
        return out_f32

    def forward(self, x_to_upsample, x):
        y = self.forward_hl(dense.from_f32(x_to_upsample.unsqueeze(1)), x)
        return dense.to_f32(y, 0, self.out_channels).squeeze(1)
