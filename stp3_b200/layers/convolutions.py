"""2-D building blocks of the BEV path with the reference's constructor signatures and parameter names
(stp3/layers/convolutions.py:183-280) so checkpoints load unchanged; forward() runs on the wgmma kernels.

  UpsamplingAdd  : bilinear x2 -> 1x1 conv -> BN, + skip.   Executed as 1x1 conv + folded BN at LOW resolution and a
                   fused upsample+add kernel (the interpolation weights sum to one, so the affine map commutes).
  ASPP / DeepLabHead : the five ASPP branches write straight into one channels-last concat tensor; the global-pool
                   branch is spatially constant and becomes a per-image bias of the 1x1 projection.  DeepLabHead also
                   runs in train() (batch statistics, dropout, autograd; dense_train.py).
  UpsamplingConcat : bilinear x2 of the coarse map into its channel window of the concat tensor, two 3x3 conv/BN/ReLU;
                   also in train().
  Bottleneck / LayerNorm / Block / Bottleblock : the prediction stage's blocks, eval only (DESIGN.md §3.16); the
                   planner's channel reduction uses Bottleneck too (§3.17).
"""
import os
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .. import dense, dense_train
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
        """x (N,Cin,H,W) fp32 -> (N,num_classes,H,W) fp32.  In train mode every BatchNorm uses batch statistics (and
        updates its running ones), the projection's Dropout draws its mask from torch's default generator, and the output
        carries a grad_fn whose backward fills every parameter's .grad (and x's, when x requires grad)."""
        if self.training:
            return self._forward_train(x)
        y = self.forward_hl(dense.from_f32(x.unsqueeze(1)))
        return dense.to_f32(y, 0, self.num_classes).squeeze(1)

    # ------------------------------------------------------------------------------------------------ train mode
    def _forward_train(self, x: torch.Tensor) -> torch.Tensor:
        for name, m in self.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                dense_train.check_bn(m, f"DeepLabHead.{name}")
        if not x.is_cuda or not self[1].weight.is_cuda:
            raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
        if x.dim() != 4 or x.shape[1] != self.in_channels:
            raise ValueError(f"DeepLabHead: expected (N, {self.in_channels}, H, W), got {tuple(x.shape)}")
        if x.shape[0] * dense_train.sync_world(self[0].convs[-1][2], x.shape[0], "DeepLabHead") < 2:
            # the pooling branch's BatchNorm sees one value per image and channel (nn.BatchNorm2d raises the same);
            # under SyncBatchNorm it sees the process group's images
            raise ValueError("DeepLabHead (train mode): Expected more than 1 value per channel when training, got input "
                             f"size {(x.shape[0], self.hidden, 1, 1)} in the ASPP pooling branch")
        return _DeepLabTrainFn.apply(self, x.float(), *self.parameters())

    def _train_forward(self, x: torch.Tensor):
        """x (N, Cin, H, W) fp32 -> (logits (N, num_classes, H, W), tape for _train_backward)."""
        aspp: ASPP = self[0]
        h, nb = self.hidden, 1 + len(aspp.rates)
        N, cin, H, W = x.shape
        dev = x.device
        x_cl = x.detach().permute(0, 2, 3, 1).contiguous()
        mode = dense_train.amp_mode()
        x_hl = dense_train.to_hl(x_cl, **dense_train.amp_kw(mode))
        # the nb spatial branches write their activated outputs side by side: the projection's input
        cat = torch.empty((N, H, W, nb * h), dtype=torch.float32, device=dev)
        branches = []
        for i in range(nb):
            conv, bn = aspp.convs[i][0], aspp.convs[i][1]
            raw = dense_train.conv_raw(x_hl, conv.weight, 1, dilation=conv.dilation[0])
            st = dense_train.bn_stats_module(raw, bn)
            dense_train.bn_apply(raw, st, bn.weight, bn.bias, relu=True, hl=False, y_out=cat[..., i * h:(i + 1) * h])
            branches.append((conv, bn, raw, st))
        # global-pool branch: per-image means -> 1x1 -> BatchNorm over the N images -> ReLU; spatially constant, so it
        # enters the projection as a per-image bias and the broadcast map is never built
        pconv, pbn = aspp.convs[nb][1], aspp.convs[nb][2]
        mean = dense_train.image_channel_sums(x_cl) * (1.0 / (H * W))
        v_raw = torch.empty((N, 1, 1, h), dtype=torch.float32, device=dev)
        dense.small_linear(mean, pconv.weight.detach().float().reshape(h, cin).contiguous(), v_raw.view(N, h), False)
        pst = dense_train.bn_stats_module(v_raw, pbn)
        v, _ = dense_train.bn_apply(v_raw, pst, pbn.weight, pbn.bias, relu=True, hl=False)
        proj, proj_bn, drop = aspp.project[0], aspp.project[1], aspp.project[3]
        w_proj = proj.weight.detach().float().reshape(h, (nb + 1) * h)
        pbias = torch.zeros((N, dense.out_tile(h)), dtype=torch.float32, device=dev)
        dense.small_linear(v.view(N, h), w_proj[:, nb * h:].contiguous(), pbias, False)
        praw = dense_train.conv_raw(dense_train.to_hl(cat, **dense_train.amp_kw(mode)), w_proj[:, :nb * h].reshape(h, nb * h, 1, 1), 1,
                                    img_bias=pbias)
        proj_st = dense_train.bn_stats_module(praw, proj_bn)
        p = float(drop.p) if drop.training else 0.0
        seed = int(torch.randint(0, 2 ** 63 - 1, (1,)).item()) if p > 0 else 0     # torch.manual_seed reproduces it
        z, z_hl = dense_train.bn_apply(praw, proj_st, proj_bn.weight, proj_bn.bias, relu=True, dropout=(p, seed, 0),
                                       **dense_train.amp_kw(mode))
        raw3 = dense_train.conv_raw(z_hl, self[1].weight, 1)
        st3 = dense_train.bn_stats_module(raw3, self[2])
        y3, y3_hl = dense_train.bn_apply(raw3, st3, self[2].weight, self[2].bias, relu=True, **dense_train.amp_kw(mode))
        out = dense_train.conv_raw(y3_hl, self[4].weight, 1, bias=self[4].bias, nchw=True)
        # x: what the branches' weight gradients read (under autocast the plane they multiplied, not an fp32 copy)
        tape = {"x": x_cl if mode is None else x_hl, "shape": (N, H, W, cin), "cat": cat, "branches": branches, "mean": mean, "v_raw": v_raw, "pst": pst, "v": v,
                "praw": praw, "proj_st": proj_st, "p": p, "z": z, "raw3": raw3, "st3": st3, "y3": y3, "mode": mode}
        return out, tape

    def _train_backward(self, tape, g_out: torch.Tensor, need_x: bool):
        """Reverse walk of _train_forward -> (dL/dx (N, Cin, H, W) or None, {parameter: gradient})."""
        aspp: ASPP = self[0]
        h, nb = self.hidden, 1 + len(aspp.rates)
        x_op = tape["x"]
        N, H, W, cin = tape["shape"]
        dev = tape["cat"].device
        grads = {}
        mode = tape["mode"]       # the spatial convolutions' precision; the pooling branch's products stay fp32
        op = lambda t: dense_train.operand(t, mode)     # noqa: E731  (one plane per gradient under autocast)
        conv3, bn3, cls = self[1], self[2], self[4]
        g = g_out.float().permute(0, 2, 3, 1).contiguous()
        grads[cls.bias] = dense_train.channel_sums(g)
        g_op = op(g)
        grads[cls.weight] = dense_train.conv_wgrad(tape["y3"], g_op, 1, 1, 1, **dense_train.amp_kw(mode))
        g = dense_train.conv_dgrad(g_op, cls.weight, 1, H, W, **dense_train.amp_kw(mode))
        g, grads[bn3.weight], grads[bn3.bias], _ = dense_train.bn_backward(g, tape["raw3"], tape["st3"], bn3.weight,
                                                                          tape["y3"])
        g_op = op(g)
        grads[conv3.weight] = dense_train.conv_wgrad(tape["z"], g_op, 3, 3, 1, **dense_train.amp_kw(mode))
        # dropout: z > 0 marks the kept positive elements (the projection BN's mask below); the 1 / (1 - p) factor of
        # the kept ones rides on the transposed 3x3 weights
        p = tape["p"]
        w3 = conv3.weight.detach().float() * (1.0 / (1.0 - p)) if p > 0 else conv3.weight
        g = dense_train.conv_dgrad(g_op, w3, 1, H, W, **dense_train.amp_kw(mode))
        proj, proj_bn = aspp.project[0], aspp.project[1]
        g, grads[proj_bn.weight], grads[proj_bn.bias], _ = dense_train.bn_backward(g, tape["praw"], tape["proj_st"],
                                                                                  proj_bn.weight, tape["z"])
        # projection: the spatial branches' columns from the concat tensor, the pooled ones from the per-image sums of g
        w_proj = proj.weight.detach().float().reshape(h, (nb + 1) * h)
        gsum = dense_train.image_channel_sums(g)
        dw_pool = dense_train.conv_wgrad(tape["v"], gsum.view(N, 1, 1, h), 1, 1, 1)
        g_op = op(g)
        grads[proj.weight] = torch.cat([dense_train.conv_wgrad(tape["cat"], g_op, 1, 1, 1, **dense_train.amp_kw(mode)),
                                        dw_pool], dim=1)
        g_v = torch.empty((N, 1, 1, h), dtype=torch.float32, device=dev)
        dense.small_linear(gsum, w_proj[:, nb * h:].t().contiguous(), g_v.view(N, h), False)
        pconv, pbn = aspp.convs[nb][1], aspp.convs[nb][2]
        g_v, grads[pbn.weight], grads[pbn.bias], _ = dense_train.bn_backward(g_v, tape["v_raw"], tape["pst"],
                                                                            pbn.weight, tape["v"])
        grads[pconv.weight] = dense_train.conv_wgrad(tape["mean"].view(N, 1, 1, cin), g_v, 1, 1, 1)
        gx = None
        if need_x:
            # the pooled branch's input gradient, W1^T g_v / (H W) per image, is added by the first branch's dgrad
            # epilogue as its per-image bias
            w1t = pconv.weight.detach().float().reshape(h, cin).t() * (1.0 / (H * W))
            gx_pool = torch.zeros((N, dense.out_tile(cin)), dtype=torch.float32, device=dev)
            dense.small_linear(g_v.view(N, h), w1t.contiguous(), gx_pool, False)
        for i, (conv, bn, raw, st) in enumerate(tape["branches"]):
            sl = slice(i * h, (i + 1) * h)
            gb = dense_train.conv_dgrad(g_op, w_proj[:, sl].reshape(h, h, 1, 1), 1, H, W, **dense_train.amp_kw(mode))
            gb, grads[bn.weight], grads[bn.bias], _ = dense_train.bn_backward(gb, raw, st, bn.weight,
                                                                             tape["cat"][..., sl])
            k, d = conv.kernel_size[0], conv.dilation[0]
            gb_op = op(gb)
            grads[conv.weight] = dense_train.conv_wgrad(x_op, gb_op, k, k, 1, dilation=d, **dense_train.amp_kw(mode))
            if need_x:
                gxi = dense_train.conv_dgrad(gb_op, conv.weight, 1, H, W, dilation=d,
                                             img_bias=gx_pool if i == 0 else None, **dense_train.amp_kw(mode))
                gx = gxi if gx is None else gx.add_(gxi)
        return (gx.permute(0, 3, 1, 2).contiguous() if need_x else None), grads


class _DeepLabTrainFn(torch.autograd.Function):
    """The train-mode DeepLab head as one autograd node, like the decoder's (_DecoderTrainFn): forward keeps the
    activations and statistics, backward walks the layers in reverse on the train-mode kernels.  The backward is not
    itself differentiable, runs once per forward (retain_graph is refused), and refuses weights modified in place
    between forward and backward."""

    @staticmethod
    def forward(ctx, head, x, *params):
        out, tape = head._train_forward(x)
        ctx.head, ctx.tape, ctx.params = head, tape, params
        ctx.versions = [p._version for p in params]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        if ctx.tape is None:
            raise RuntimeError("DeepLabHead (train mode): backward ran a second time through the same forward; the "
                               "activations are released after the first backward (retain_graph is not supported) -- "
                               "run the forward again")
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("DeepLabHead (train mode): a head parameter was modified in place between forward and "
                               "backward (e.g. optimizer.step() before loss.backward())")
        tape, ctx.tape = ctx.tape, None
        gx, grads = ctx.head._train_backward(tape, g_out, ctx.needs_input_grad[1])
        return (None, gx) + tuple(grads.get(p) for p in ctx.params)


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
        return self._convs(cat, P[key], out_f32, out_f32_nhwc)

    def forward_cat(self, coarse: dense.HL, cat: dense.HL, cf: int, out_f32: Optional[torch.Tensor] = None,
                    out_f32_nhwc: bool = False):
        """forward_hl with the fine map already in channels [0, cf) of `cat` (B, 1, 2h, 2w, pad_to(cf + coarse.c)) hi/lo,
        where its producer wrote it: the upsampled coarse map goes into the channels behind it, so the fine map makes no
        fp32 round trip.  The other channels of `cat` need not be initialised."""
        self._require_eval()
        P = self.packed()
        cc = coarse.c
        assert cf + cc == self.in_channels and cf % 8 == 0 and cat.hi.shape[-1] == dense.pad_to(cf + cc)
        key = ("c0p", cf, cc)
        if key not in P:
            P[key] = dense.pack_conv(P["c0"][0], P["c0"][1], in_layout=[(0, cf, 0), (cf, cc, cf)])
        # the first convolution reads channels up to k_hi: the coarse map's zero padding channels fill the gap
        n_up = (P[key].k_hi or cat.hi.shape[-1]) - cf
        assert n_up <= coarse.hi.shape[-1]
        dense.upsample2x_add(coarse, None, n_up, out=cat, out_coff=cf)
        return self._convs(cat, P[key], out_f32, out_f32_nhwc)

    def _convs(self, cat: dense.HL, pc0: dense.PackedConv, out_f32, out_f32_nhwc):
        P = self.packed()
        y = dense.conv(cat, pc0, relu=True)
        if out_f32 is None:
            return dense.conv(y, P["c1"], relu=True)
        B = y.hi.shape[0]
        shape = (B, *y.hi.shape[2:4], self.out_channels) if out_f32_nhwc else (B, self.out_channels, *y.hi.shape[2:4])
        assert tuple(out_f32.shape) == shape and out_f32.dtype == torch.float32 and out_f32.is_contiguous()
        dense.conv(y, P["c1"], relu=True, out_f32=out_f32, n_valid=self.out_channels, out_f32_nhwc=out_f32_nhwc, store=False)
        return out_f32

    def forward(self, x_to_upsample, x, channels_last: bool = False):
        """x_to_upsample (N,Cc,h,w), x (N,Cf,2h,2w) fp32 -> (N,Cout,2h,2w) like the reference module.  In train mode
        both BatchNorms use batch statistics (and update their running ones) and the output carries a grad_fn whose
        backward fills the four parameters' .grad and the gradients of the inputs that require one; channels_last
        (train mode only) returns (N,2h,2w,Cout) and takes its gradient in that layout -- what the lift-splat reads and
        its backward writes, so the encoder's train path transposes neither."""
        if self.training:
            return self._forward_train(x_to_upsample, x, channels_last)
        if channels_last:
            raise ValueError("UpsamplingConcat.forward: channels_last is the train path's; in eval mode use forward_hl("
                             "out_f32=..., out_f32_nhwc=True)")
        y = self.forward_hl(dense.from_f32(x_to_upsample.unsqueeze(1)), x)
        return dense.to_f32(y, 0, self.out_channels).squeeze(1)

    # ------------------------------------------------------------------------------------------------ train mode
    def _forward_train(self, x_up: torch.Tensor, x: torch.Tensor, channels_last: bool) -> torch.Tensor:
        for i in (1, 4):
            dense_train.check_bn(self.conv[i], f"UpsamplingConcat.conv.{i}")
        if not x.is_cuda or not x_up.is_cuda or not self.conv[0].weight.is_cuda:
            raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
        if x.dim() != 4 or x_up.dim() != 4 or x.shape[1] + x_up.shape[1] != self.in_channels or \
                x.shape[0] != x_up.shape[0] or tuple(x.shape[2:]) != (2 * x_up.shape[2], 2 * x_up.shape[3]):
            raise ValueError(f"UpsamplingConcat: expected (N, Cc, h, w) and (N, {self.in_channels} - Cc, 2h, 2w), got "
                             f"{tuple(x_up.shape)} and {tuple(x.shape)}")
        dense_train.sync_world(self.conv[1], x.shape[0], "UpsamplingConcat")
        return _UpsamplingConcatTrainFn.apply(self, x_up.float(), x.float(), channels_last, *self.parameters())

    def _train_forward(self, x_up: torch.Tensor, x: torch.Tensor, channels_last: bool):
        """-> (output (N, Cout, 2h, 2w), or (N, 2h, 2w, Cout) with channels_last; tape for _train_backward)."""
        N, cf, H, W = x.shape
        cc = x_up.shape[1]
        # the concat tensor [fine | upsampled coarse], channels-last: the fine map is copied into its window, the
        # upsample kernel writes the coarse map's
        cat = torch.empty((N, H, W, cf + cc), dtype=torch.float32, device=x.device)
        cat[..., :cf].copy_(x.detach().permute(0, 2, 3, 1))
        dense_train.upsample2x_into(x_up.detach().permute(0, 2, 3, 1).contiguous(), cat, cf)
        conv0, bn0, conv1, bn1 = self.conv[0], self.conv[1], self.conv[3], self.conv[4]
        mode = dense_train.amp_mode()
        cat_hl = dense_train.to_hl(cat, **dense_train.amp_kw(mode))
        raw0 = dense_train.conv_raw(cat_hl, conv0.weight, 1)
        st0 = dense_train.bn_stats_module(raw0, bn0)
        y0, y0_hl = dense_train.bn_apply(raw0, st0, bn0.weight, bn0.bias, relu=True, **dense_train.amp_kw(mode))
        raw1 = dense_train.conv_raw(y0_hl, conv1.weight, 1)
        st1 = dense_train.bn_stats_module(raw1, bn1)
        y1, _ = dense_train.bn_apply(raw1, st1, bn1.weight, bn1.bias, relu=True, hl=False)
        # cat: what conv0's weight gradient reads (under autocast the plane it multiplied, not an fp32 copy)
        tape = {"cat": cat if mode is None else cat_hl, "shape": tuple(cat.shape), "cf": cf, "raw0": raw0, "st0": st0,
                "y0": y0, "raw1": raw1, "st1": st1, "y1": y1, "mode": mode}
        return (y1 if channels_last else y1.permute(0, 3, 1, 2).contiguous()), tape

    def _train_backward(self, tape, g_out: torch.Tensor, channels_last: bool, need_up: bool, need_x: bool):
        """Reverse walk of _train_forward -> (dL/dx_to_upsample or None, dL/dx or None (both NCHW), {parameter: gradient})."""
        conv0, bn0, conv1, bn1 = self.conv[0], self.conv[1], self.conv[3], self.conv[4]
        cat, cf = tape["cat"], tape["cf"]
        N, H, W, ccat = tape["shape"]
        grads = {}
        g = g_out.float().contiguous() if channels_last else g_out.float().permute(0, 2, 3, 1).contiguous()
        g, grads[bn1.weight], grads[bn1.bias], _ = dense_train.bn_backward(g, tape["raw1"], tape["st1"], bn1.weight,
                                                                          tape["y1"])
        mode = tape["mode"]
        g_op = dense_train.operand(g, mode)                # one plane for both products under autocast
        grads[conv1.weight] = dense_train.conv_wgrad(tape["y0"], g_op, 3, 3, 1, **dense_train.amp_kw(mode))
        g = dense_train.conv_dgrad(g_op, conv1.weight, 1, H, W, **dense_train.amp_kw(mode))
        g, grads[bn0.weight], grads[bn0.bias], _ = dense_train.bn_backward(g, tape["raw0"], tape["st0"], bn0.weight,
                                                                          tape["y0"])
        g_op = dense_train.operand(g, mode)
        grads[conv0.weight] = dense_train.conv_wgrad(cat, g_op, 3, 3, 1, **dense_train.amp_kw(mode))
        g_up = g_x = None
        if need_up or need_x:
            # the concat gradient splits: the fine map's channels as they are, the coarse map's through the adjoint of
            # the upsample, read from their window
            g_cat = dense_train.conv_dgrad(g_op, conv0.weight, 1, H, W, **dense_train.amp_kw(mode))
            if need_x:
                g_x = g_cat[..., :cf].permute(0, 3, 1, 2).contiguous()
            if need_up:
                g_up = dense_train.upsample2x_backward_from(g_cat, cf, ccat - cf).permute(0, 3, 1, 2).contiguous()
        return g_up, g_x, grads


class _UpsamplingConcatTrainFn(torch.autograd.Function):
    """UpsamplingConcat in train mode as one autograd node, with the guards of _DeepLabTrainFn: the backward is not
    itself differentiable, runs once per forward, and refuses parameters modified in place in between."""

    @staticmethod
    def forward(ctx, mod, x_up, x, channels_last, *params):
        out, tape = mod._train_forward(x_up, x, channels_last)
        ctx.mod, ctx.tape, ctx.params, ctx.channels_last = mod, tape, params, channels_last
        ctx.versions = [p._version for p in params]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        if ctx.tape is None:
            raise RuntimeError("UpsamplingConcat (train mode): backward ran a second time through the same forward; the "
                               "activations are released after the first backward (retain_graph is not supported) -- "
                               "run the forward again")
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("UpsamplingConcat (train mode): a parameter was modified in place between forward and "
                               "backward (e.g. optimizer.step() before loss.backward())")
        tape, ctx.tape = ctx.tape, None
        g_up, g_x, grads = ctx.mod._train_backward(tape, g_out, ctx.channels_last, ctx.needs_input_grad[1],
                                                   ctx.needs_input_grad[2])
        return (None, g_up, g_x, None) + tuple(grads.get(p) for p in ctx.params)


# ------------------------------------------------------------------------------------------------ prediction stage
# Eval-only modules of the future-prediction stage (convolutions.py:65-170, 283-380).  Their convolutions run on
# stp3_conv_fwd; LayerNorm, GELU, the depthwise 7x7 and the skip's max pool on the per-pixel kernels of
# predict_kernels.cu.
PREDICT_EVAL_ONLY = ("the prediction stage (N_FUTURE_FRAMES > 0) is eval-only on sm_90a: its gradients, the train-time "
                     "noise and the probabilistic loss are not implemented -- call .eval()")


class PredictModule(PackedModule):
    def _require_eval(self):
        if any(m.training for m in self.modules()):
            raise NotImplementedError(f"{type(self).__name__}: {PREDICT_EVAL_ONLY}")

    def forward(self, x):
        """x (N, C, H, W) fp32 on the device -> (N, C_out, H, W') fp32 through forward_hl."""
        y = self.forward_hl(dense.from_f32(x.unsqueeze(1)))
        return dense.to_f32(y).squeeze(1)


def _ln_params(ln):
    return (ln.weight.detach().float().contiguous(), ln.bias.detach().float().contiguous(), float(ln.eps))


class LayerNorm(nn.Module):
    """The reference's LayerNorm (convolutions.py:283-306): parameters `weight` / `bias` over C channels, eps 1e-6,
    biased variance.  Both data formats normalise each pixel's channel vector, which is what stp3_channel_norm_act and
    stp3_dw_ln compute; inside Block and Bottleblock the parent runs it fused with its neighbours.  Called on its own it
    runs stp3_channel_norm_act, eval only, for C <= 256 channels (a multiple of 8)."""

    def __init__(self, normalized_shape, eps=1e-6, data_format="channels_last"):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps
        self.data_format = data_format
        if self.data_format not in ["channels_last", "channels_first"]:
            raise NotImplementedError
        self.normalized_shape = (normalized_shape,)

    def forward(self, x):
        """channels_first: x (N, C, H, W); channels_last: x (..., C); fp32 on the device, same shape out."""
        if self.training:
            raise NotImplementedError(f"LayerNorm: {PREDICT_EVAL_ONLY}")
        C = self.normalized_shape[0]
        if C % 8 != 0 or C > 256:
            raise NotImplementedError(f"LayerNorm over {C} channels: stp3_channel_norm_act takes a multiple of 8, at "
                                      "most 256")
        if self.data_format == "channels_last":                     # one image of numel / C pixels
            h = dense.from_f32(x.reshape(1, 1, -1, 1, C), channels_last=True)
            dense.channel_norm_act(h, h, C, ln=_ln_params(self))
            return dense.to_f32(h, 0, C)[0, 0, :, :, 0].t().reshape(x.shape)
        h = dense.from_f32(x.reshape(1, -1, C, *x.shape[-2:]))      # N images
        dense.channel_norm_act(h, h, C, ln=_ln_params(self))
        return dense.to_f32(h, 0, C).reshape(x.shape)


class Bottleneck(PredictModule):
    """The reference's Bottleneck (convolutions.py:65-170) in the two forms the reference configurations build:
      downsample=True (the present distribution and the planner's first three blocks): 1x1 -> BN -> ReLU -> 3x3 s2 ->
        BN -> ReLU -> 1x1 -> BN -> ReLU, plus the skip (zero-pad an odd H / W, MaxPool 2x2, 1x1 -> BN);
      out_channels != in_channels without resampling (the planner's last block, Bottleneck(32, 8)): the same with a
        stride-1 3x3 and the skip 1x1 -> BN of the input, no pool.
    The skip is the up-projection's residual, added after its ReLU."""

    def __init__(self, in_channels, out_channels=None, kernel_size=3, dilation=1, groups=1, upsample=False,
                 downsample=False, dropout=0.0):
        super().__init__()
        out_channels = out_channels or in_channels
        if upsample or kernel_size != 3 or dilation != 1 or groups != 1 or (not downsample and out_channels == in_channels):
            raise NotImplementedError("Bottleneck: only the downsampling 3x3 form (the present distribution's) and the "
                                      "projecting stride-1 3x3 form (the planner's last block) are built")
        self._downsample = downsample
        bottleneck_channels = int(in_channels / 2)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.layers = nn.Sequential(OrderedDict([
            ('conv_down_project', nn.Conv2d(in_channels, bottleneck_channels, kernel_size=1, bias=False)),
            ('abn_down_project', nn.Sequential(nn.BatchNorm2d(bottleneck_channels), nn.ReLU(inplace=True))),
            ('conv', nn.Conv2d(bottleneck_channels, bottleneck_channels, kernel_size=3, bias=False,
                               stride=2 if downsample else 1, padding=1)),
            ('abn', nn.Sequential(nn.BatchNorm2d(bottleneck_channels), nn.ReLU(inplace=True))),
            ('conv_up_project', nn.Conv2d(bottleneck_channels, out_channels, kernel_size=1, bias=False)),
            ('abn_up_project', nn.Sequential(nn.BatchNorm2d(out_channels), nn.ReLU(inplace=True))),
            ('dropout', nn.Dropout2d(p=dropout)),
        ]))
        projection = OrderedDict()
        if downsample:
            projection['upsample_skip_proj'] = nn.MaxPool2d(kernel_size=2, stride=2)
        projection['conv_skip_proj'] = nn.Conv2d(in_channels, out_channels, kernel_size=1, bias=False)
        projection['bn_skip_proj'] = nn.BatchNorm2d(out_channels)
        self.projection = nn.Sequential(projection)

    def _pack(self):
        L = self.layers
        P = {}
        for key, conv, bn in (("down", L.conv_down_project, L.abn_down_project[0]), ("conv", L.conv, L.abn[0]),
                              ("up", L.conv_up_project, L.abn_up_project[0]),
                              ("skip", self.projection.conv_skip_proj, self.projection.bn_skip_proj)):
            w, b = dense.fold_bn(conv.weight, bn)
            P[key] = dense.pack_conv(w, b, stride=conv.stride[0])
        return P

    def forward_hl(self, x: dense.HL) -> dense.HL:
        """x: HL (B, T, H, W, >= in_channels) -> HL (B, T, ceil(H/2), ceil(W/2), 64-padded out_channels), or
        (B, T, H, W, ...) for the stride-1 form."""
        self._require_eval()
        P = self.packed()
        a = dense.conv(x, P["down"], relu=True)
        a = dense.conv(a, P["conv"], relu=True)
        skip = dense.conv(dense.maxpool2_pad(x) if self._downsample else x, P["skip"])
        return dense.conv(a, P["up"], relu=True, residual=skip, res_after_act=True)


class Block(PredictModule):
    """ConvNeXt Block (convolutions.py:308-345): depthwise 7x7 + bias -> LayerNorm -> Linear(C, 4C) -> GELU ->
    Linear(4C, C) -> * gamma -> + input.  gamma folds into pwconv2's weight and bias; the input is the residual of that
    convolution."""

    def __init__(self, dim, drop_path=0., layer_scale_init_value=1e-6):
        super().__init__()
        if drop_path > 0.:
            raise NotImplementedError("Block: drop_path > 0 is a training regulariser (no reference config uses it)")
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, 4 * dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(4 * dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones((dim)),
                                  requires_grad=True) if layer_scale_init_value > 0 else None
        self.drop_path = nn.Identity()
        self.dim = dim

    def _pack(self):
        C = self.dim
        g = self.gamma.detach().float() if self.gamma is not None else torch.ones(C, device=self.pwconv2.weight.device)
        w2 = self.pwconv2.weight.detach().float() * g[:, None]
        b2 = self.pwconv2.bias.detach().float() * g
        return {"dw_w": self.dwconv.weight.detach().float().reshape(C, 49).t().contiguous(),
                "dw_b": self.dwconv.bias.detach().float().contiguous(), "ln": _ln_params(self.norm),
                "pw1": dense.pack_conv(self.pwconv1.weight.detach().float().view(4 * C, C, 1, 1),
                                       self.pwconv1.bias.detach().float()),
                "pw2": dense.pack_conv(w2.view(C, 4 * C, 1, 1), b2)}

    def forward_hl(self, x: dense.HL) -> dense.HL:
        """x: HL (B, T, H, W, >= dim) -> HL (B, T, H, W, 64-padded dim)."""
        self._require_eval()
        P = self.packed()
        B, T, H, W, _ = x.hi.shape
        C = self.dim
        t = (dense.HL.empty if C % dense.KB == 0 else dense.HL.zeros)(B, T, H, W, C, x.hi.device)   # padding feeds pw1
        dense.dw_ln(x, P["dw_w"], P["dw_b"], 7, P["ln"], t, C)
        y = dense.conv(t, P["pw1"])
        dense.channel_norm_act(y, y, 4 * C, gelu=True)
        return dense.conv(y, P["pw2"], residual=x)


class Bottleblock(PredictModule):
    """The trusting gate's block (convolutions.py:347-380): 7x7 -> LN -> GELU -> 1x1 -> LN -> GELU -> 3x3 -> LN -> GELU
    (channels-first LayerNorms, no conv bias), plus GELU(1x1(x)) when the channel count changes (else x)."""

    def __init__(self, in_channels, out_channels=None):
        super().__init__()
        bottleneck_channels = int(in_channels / 2)
        out_channels = out_channels or in_channels
        self.in_channels, self.out_channels, self.mid = in_channels, out_channels, bottleneck_channels
        self.layers = nn.Sequential(
            nn.Conv2d(in_channels, bottleneck_channels, kernel_size=7, bias=False, padding=3),
            LayerNorm(bottleneck_channels, eps=1e-6, data_format='channels_first'),
            nn.GELU(),
            nn.Conv2d(bottleneck_channels, bottleneck_channels, kernel_size=1, bias=False),
            LayerNorm(bottleneck_channels, eps=1e-6, data_format='channels_first'),
            nn.GELU(),
            nn.Conv2d(bottleneck_channels, out_channels, kernel_size=3, bias=False, padding=1),
            LayerNorm(out_channels, eps=1e-6, data_format='channels_first'),
            nn.GELU()
        )
        if out_channels == in_channels:
            self.projection = None
        else:
            self.projection = nn.Sequential(nn.Conv2d(in_channels, out_channels, kernel_size=1, bias=False), nn.GELU())

    def _pack(self):
        L = self.layers
        z = lambda c: torch.zeros(c.out_channels, device=c.weight.device)
        P = {f"c{i}": dense.pack_conv(L[i].weight.detach().float(), z(L[i])) for i in (3, 6)}
        # the 7x7 runs as one launch per 64 input channels, each adding the previous one's output as its residual: one
        # launch over all 128 channels is a 6272-long sum in the wgmma accumulator, whose round-off grows with the
        # length of the sum faster than round-to-nearest fp32 adds would, to 3e-5 of max (DESIGN.md section 4)
        w0 = L[0].weight.detach().float()
        P["c0"] = [dense.pack_conv(w0[:, c:c + dense.KB].contiguous(), z(L[0])) for c in range(0, w0.shape[1], dense.KB)]
        P.update({f"ln{i}": _ln_params(L[i]) for i in (1, 4, 7)})
        if self.projection is not None:
            P["proj"] = dense.pack_conv(self.projection[0].weight.detach().float(), z(self.projection[0]))
        return P

    def forward_hl(self, x: dense.HL) -> dense.HL:
        """x: HL (B, T, H, W, >= in_channels) -> HL (B, T, H, W, 64-padded out_channels)."""
        self._require_eval()
        P = self.packed()
        m, co = self.mid, self.out_channels
        a = None
        for i, pc in enumerate(P["c0"]):
            a = dense.conv(x, pc, cin_off=i * dense.KB, residual=a)
        dense.channel_norm_act(a, a, m, ln=P["ln1"], gelu=True)
        a = dense.conv(a, P["c3"])
        dense.channel_norm_act(a, a, m, ln=P["ln4"], gelu=True)
        a = dense.conv(a, P["c6"])
        if self.projection is not None:
            y, gelu_y = dense.conv(x, P["proj"]), True
        else:
            y, gelu_y = x, False
        dense.channel_norm_act(a, a, co, ln=P["ln7"], gelu=True, y=y, gelu_y=gelu_y)
        return a
