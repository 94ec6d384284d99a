"""BEV decoder with the reference's constructor/forward surface and parameter names (stp3/models/decoder.py:8-140):
ResNet-18 stages 1-3 as a U-Net over the BEV grid and 3x3 -> 1x1 heads, executed on the wgmma kernels."""
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable
from torchvision.models.resnet import resnet18

from .. import dense, dense_train
from ..layers._packing import PackedModule
from ..layers.convolutions import UpsamplingAdd


def _head(cin, cout, sigmoid=False):
    layers = [nn.Conv2d(cin, cin, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(cin), nn.ReLU(inplace=True),
              nn.Conv2d(cin, cout, kernel_size=1, padding=0)]
    if sigmoid:
        layers.append(nn.Sigmoid())
    return nn.Sequential(*layers)


class Decoder(PackedModule):
    def __init__(self, in_channels, n_classes, n_present, n_hdmap, predict_gate):
        super().__init__()
        self.perceive_hdmap = predict_gate['perceive_hdmap']
        self.predict_pedestrian = predict_gate['predict_pedestrian']
        self.predict_instance = predict_gate['predict_instance']
        self.predict_future_flow = predict_gate['predict_future_flow']
        self.planning = predict_gate['planning']
        self.n_classes = n_classes
        self.n_present = n_present
        if self.predict_instance is False and self.predict_future_flow is True:
            raise ValueError('flow cannot be True when not predicting instance')

        backbone = resnet18(weights=None, zero_init_residual=True)
        self.first_conv = nn.Conv2d(in_channels, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = backbone.bn1
        self.relu = backbone.relu
        self.layer1, self.layer2, self.layer3 = backbone.layer1, backbone.layer2, backbone.layer3

        c = in_channels
        self.up3_skip = UpsamplingAdd(256, 128, scale_factor=2)
        self.up2_skip = UpsamplingAdd(128, 64, scale_factor=2)
        self.up1_skip = UpsamplingAdd(64, c, scale_factor=2)

        self.segmentation_head = _head(c, self.n_classes)
        if self.predict_pedestrian:
            self.pedestrian_head = _head(c, self.n_classes)
        if self.perceive_hdmap:
            self.hdmap_head = _head(c, 2 * n_hdmap)
        if self.predict_instance:
            self.instance_offset_head = _head(c, 2)
            self.instance_center_head = _head(c, 1, sigmoid=True)
        if self.predict_future_flow:
            self.instance_future_head = _head(c, 2)
        if self.planning:
            self.costvolume_head = _head(c, 1)
        self.in_channels = in_channels

    # output key -> (module attribute, present-frame only, squeeze channel)
    _HEADS = (("segmentation", "segmentation_head", False), ("pedestrian", "pedestrian_head", False),
              ("hdmap", "hdmap_head", True), ("instance_center", "instance_center_head", False),
              ("instance_offset", "instance_offset_head", False), ("instance_flow", "instance_future_head", False),
              ("costvolume", "costvolume_head", False))

    def _pack(self):
        P = {}
        w, b = dense.fold_bn(self.first_conv.weight, self.bn1)
        P["first"] = dense.pack_conv(w, b, stride=2)
        for name in ("layer1", "layer2", "layer3"):
            for i, blk in enumerate(getattr(self, name)):
                w, b = dense.fold_bn(blk.conv1.weight, blk.bn1)
                P[f"{name}.{i}.c1"] = dense.pack_conv(w, b, stride=blk.conv1.stride[0])
                w, b = dense.fold_bn(blk.conv2.weight, blk.bn2)
                P[f"{name}.{i}.c2"] = dense.pack_conv(w, b)
                if blk.downsample is not None:
                    w, b = dense.fold_bn(blk.downsample[0].weight, blk.downsample[1])
                    P[f"{name}.{i}.ds"] = dense.pack_conv(w, b, stride=blk.downsample[0].stride[0])
        # heads: the 3x3 convolutions of the all-frame heads share their input -> concatenated along N in groups of
        # <= 256 columns; every head's 1x1 conv(+bias, +sigmoid) is evaluated in the epilogue of that convolution
        c = self.in_channels
        cp = dense.pad_to(c)
        all_frames = [(k, getattr(self, attr)) for k, attr, present in self._HEADS if hasattr(self, attr) and not present]
        groups, per = [], max(1, 128 // cp)          # a fused-head convolution is at most 128 columns wide
        for i in range(0, len(all_frames), per):
            groups.append(self._pack_head_group(all_frames[i:i + per], c, cp))
        P["head_groups"] = groups
        if self.perceive_hdmap:
            P["hdmap"] = self._pack_head_group([("hdmap", self.hdmap_head)], c, cp)
        return P

    @staticmethod
    def _pack_head_group(grp, c, cp):
        dev = grp[0][1][0].weight.device
        bn = dense.out_tile(len(grp) * cp)
        wcat = torch.zeros(len(grp) * cp, c, 3, 3, device=dev)
        bcat = torch.zeros(len(grp) * cp, device=dev)
        n_out = sum(h[3].out_channels for _, h in grp)
        assert n_out <= 8
        w2 = torch.zeros(n_out, bn, device=dev)
        b2 = torch.zeros(n_out, device=dev)
        members, k, mask = [], 0, 0
        for j, (key, h) in enumerate(grp):
            w_, b_ = dense.fold_bn(h[0].weight, h[1])
            wcat[j * cp:j * cp + c], bcat[j * cp:j * cp + c] = w_, b_
            ko = h[3].out_channels
            w2[k:k + ko, j * cp:j * cp + c] = h[3].weight.detach().float().reshape(ko, c)
            b2[k:k + ko] = h[3].bias.detach().float()
            if len(h) > 4:                       # nn.Sigmoid tail (instance_center head)
                mask |= ((1 << ko) - 1) << k
            members.append((key, ko))
            k += ko
        return {"conv": dense.pack_conv(wcat, bcat, bn=bn), "w2": w2.contiguous(), "b2": b2.contiguous(),
                "members": members, "mask": mask}

    def _basic_block(self, x, P, key, has_ds):
        y = dense.conv(x, P[f"{key}.c1"], relu=True)
        res = dense.conv(x, P[f"{key}.ds"]) if has_ds else x
        return dense.conv(y, P[f"{key}.c2"], relu=True, residual=res)       # relu(bn2(conv2) + identity)

    def forward_hl(self, x: dense.HL):
        if self.training:
            return self._forward_train(dense.to_f32(x))
        self._require_eval()
        P = self.packed()
        B, S, H, W, _ = x.hi.shape
        dev = x.hi.device
        skip1 = x
        y = dense.conv(x, P["first"], relu=True)
        for i, blk in enumerate(self.layer1):
            y = self._basic_block(y, P, f"layer1.{i}", blk.downsample is not None)
        skip2 = y
        for i, blk in enumerate(self.layer2):
            y = self._basic_block(y, P, f"layer2.{i}", blk.downsample is not None)
        skip3 = y
        for i, blk in enumerate(self.layer3):
            y = self._basic_block(y, P, f"layer3.{i}", blk.downsample is not None)
        y = self.up3_skip.forward_hl(y, skip3)
        y = self.up2_skip.forward_hl(y, skip2)
        y = self.up1_skip.forward_hl(y, skip1)

        out = {k: None for k, _, _ in self._HEADS}

        def run_group(G, frames, n_img):
            outs, tensors = [], {}
            for key, ko in G["members"]:
                t = torch.empty((n_img, ko, H, W), dtype=torch.float32, device=dev)
                tensors[key] = t
                outs += [(t, ch) for ch in range(ko)]
            dense.conv(y, G["conv"], relu=True, frames=frames, store=False,
                       head={"w": G["w2"], "b": G["b2"], "outs": outs, "sigmoid_mask": G["mask"]})
            return tensors

        for G in P["head_groups"]:
            for key, t in run_group(G, None, B * S).items():
                out[key] = t.view(B, S, t.shape[1], H, W)
        if self.perceive_hdmap:
            out["hdmap"] = run_group(P["hdmap"], (self.n_present - 1, 1), B)["hdmap"]
        if out["costvolume"] is not None:
            out["costvolume"] = out["costvolume"].squeeze(2)
        return out

    def forward(self, x):
        """x (B, S, C, H, W) fp32 -> dict of logits with the reference's keys and shapes (decoder.py:122-140).
        In train mode BatchNorm uses batch statistics (and updates the running ones) and the outputs carry a grad_fn
        whose backward fills the parameters' .grad (and x's, when x requires grad)."""
        if self.training:
            return self._forward_train(x)
        return self.forward_hl(dense.from_f32(x))

    # ------------------------------------------------------------------------------------------------ train mode
    def _heads(self):
        return [(key, getattr(self, attr), present) for key, attr, present in self._HEADS if hasattr(self, attr)]

    def _check_train(self):
        for name, m in self.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                dense_train.check_bn(m, f"Decoder.{name}")
        if not torch.is_tensor(self.first_conv.weight) or not self.first_conv.weight.is_cuda:
            raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")

    def _forward_train(self, x: torch.Tensor):
        self._check_train()
        bn = next(m for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm))
        dense_train.sync_world(bn, x.shape[0], "Decoder")
        x = x.float()
        params = [p for p in self.parameters()]
        keys = [k for k, _, _ in self._heads()]
        outs = _DecoderTrainFn.apply(self, x, *params)
        out = {k: None for k, _, _ in self._HEADS}
        B, S = x.shape[:2]
        for k, t in zip(keys, outs):
            out[k] = t if k == "hdmap" else t.view(B, S, *t.shape[1:])
        if out["costvolume"] is not None:
            out["costvolume"] = out["costvolume"].squeeze(2)
        return out

    @staticmethod
    def _cbn(inp, inp_hl, conv, bn, relu, res=None, hl=True, mode=None):
        """conv (no bias) -> BatchNorm with batch statistics (running ones updated) -> (+ res) -> relu?"""
        raw = dense_train.conv_raw(inp_hl, conv.weight, conv.stride[0])
        st = dense_train.bn_stats_module(raw, bn)
        y, y_hl = dense_train.bn_apply(raw, st, bn.weight, bn.bias, relu, res, hl=hl, **dense_train.amp_kw(mode))
        return y, y_hl, {"inp": inp, "hw": tuple(inp.shape[1:3]), "conv": conv, "bn": bn, "raw": raw, "st": st, "y": y,
                         "relu": relu, "mode": mode}

    @staticmethod
    def _cbn_backward(rec, g, grads, need_input=True, want_masked=False):
        """-> (dL/d inp or None, g masked by the ReLU or None); parameter gradients go to `grads`."""
        conv, bn = rec["conv"], rec["bn"]
        g_raw, dgamma, dbeta, gm = dense_train.bn_backward(g, rec["raw"], rec["st"], bn.weight,
                                                           rec["y"] if rec["relu"] else None, want_masked)
        grads[bn.weight], grads[bn.bias] = dgamma, dbeta
        kh, kw = conv.kernel_size
        mode = rec["mode"]
        g_op = dense_train.operand(g_raw, mode)           # one plane for both products under autocast
        grads[conv.weight] = dense_train.conv_wgrad(rec["inp"], g_op, kh, kw, conv.stride[0], **dense_train.amp_kw(mode))
        gin = None
        if need_input:
            gin = dense_train.conv_dgrad(g_op, conv.weight, conv.stride[0], *rec["hw"], **dense_train.amp_kw(mode))
        return gin, gm

    def _train_forward(self, x: torch.Tensor):
        """x (B, S, C, H, W) fp32 -> (head outputs in _heads() order, tape for _train_backward)."""
        B, S, C, H, W = x.shape
        N = B * S
        x_cl = x.detach().permute(0, 1, 3, 4, 2).reshape(N, H, W, C).contiguous()
        mode = dense_train.amp_mode()
        x_hl = dense_train.to_hl(x_cl, **dense_train.amp_kw(mode))
        tape = {"shape": (B, S, C, H, W), "x": x_cl, "blocks": [], "ups": [], "heads": [], "mode": mode}
        y, y_hl, tape["first"] = self._cbn(x_cl, x_hl, self.first_conv, self.bn1, relu=True, mode=mode)
        if mode is not None:      # only the first convolution's weight gradient reads the input: keep its plane
            tape["first"]["inp"] = x_hl
            tape["x"] = None
        skips = []
        for name in ("layer1", "layer2", "layer3"):
            for blk in getattr(self, name):
                r1 = r2 = rd = None
                y1, y1_hl, r1 = self._cbn(y, y_hl, blk.conv1, blk.bn1, relu=True, mode=mode)
                res = y
                if blk.downsample is not None:
                    res, _, rd = self._cbn(y, y_hl, blk.downsample[0], blk.downsample[1], relu=False, hl=False,
                                           mode=mode)
                y, y_hl, r2 = self._cbn(y1, y1_hl, blk.conv2, blk.bn2, relu=True, res=res, mode=mode)
                tape["blocks"].append((name, r1, r2, rd))
            skips.append(y)
        # UpsamplingAdd: BN(conv1x1(up(x))) + skip == BN_{stats of up(conv1x1(x))}(up(conv1x1(x))) + skip: the 1x1 runs
        # at low resolution, the statistics over the upsampled map
        for up, skip in ((self.up3_skip, skips[1]), (self.up2_skip, skips[0]), (self.up1_skip, x_cl)):
            conv, bn = up.upsample_layer[1], up.upsample_layer[2]
            low = dense_train.conv_raw(y_hl, conv.weight, 1)
            raw = dense_train.upsample2x(low)
            st = dense_train.bn_stats_module(raw, bn)
            out, y_hl = dense_train.bn_apply(raw, st, bn.weight, bn.bias, relu=False, res=skip, **dense_train.amp_kw(mode))
            tape["ups"].append({"inp": y, "conv": conv, "bn": bn, "raw": raw, "st": st})
            y = out
        outs = []
        t_present = self.n_present - 1
        for key, h, present in self._heads():
            inp, inp_hl = y, y_hl
            if present:       # the hdmap head sees the present frame only (decoder.py:134)
                Hh, Wh, c = y.shape[1:]
                inp = y.view(B, S, Hh, Wh, c)[:, t_present].contiguous()
                cp = y_hl.hi.shape[-1]
                inp_hl = dense.HL(y_hl.hi.view(B, S, 1, Hh, Wh, cp)[:, t_present].contiguous(),
                                  y_hl.lo.view(B, S, 1, Hh, Wh, cp)[:, t_present].contiguous() if y_hl.lo is not None
                                  else None, y_hl.c)
            z, z_hl, rec = self._cbn(inp, inp_hl, h[0], h[1], relu=True, mode=mode)
            sig = len(h) > 4
            o = dense_train.conv_raw(z_hl, h[3].weight, 1, bias=h[3].bias, sigmoid=sig, nchw=True)
            tape["heads"].append({"rec": rec, "conv": h[3], "z": z, "out": o, "sigmoid": sig, "present": present})
            outs.append(o)
        tape["y"] = y
        return outs, tape

    def _train_backward(self, tape, grads_out, need_x):
        """Reverse walk of _train_forward -> (dL/dx (B, S, C, H, W) or None, {parameter: gradient})."""
        B, S, C, H, W = tape["shape"]
        mode = tape["mode"]
        grads = {}
        y = tape["y"]
        g = torch.zeros_like(y)
        t_present = self.n_present - 1
        for hd, go in zip(tape["heads"], grads_out):
            go = go.contiguous().float() if go is not None else torch.zeros_like(hd["out"])
            if hd["sigmoid"]:
                go = dense_train.sigmoid_backward(go, hd["out"])
            g_cl = go.permute(0, 2, 3, 1).contiguous()                      # (n, H, W, ko)
            conv = hd["conv"]
            grads[conv.bias] = dense_train.channel_sums(g_cl)
            g_op = dense_train.operand(g_cl, mode)
            grads[conv.weight] = dense_train.conv_wgrad(hd["z"], g_op, 1, 1, 1, **dense_train.amp_kw(mode))
            gz = dense_train.conv_dgrad(g_op, conv.weight, 1, *hd["z"].shape[1:3], **dense_train.amp_kw(mode))
            gin, _ = self._cbn_backward(hd["rec"], gz, grads)
            if hd["present"]:
                g.view(B, S, *g.shape[1:])[:, t_present] += gin
            else:
                g += gin
        g_x = None
        skip_grads = []
        for u in reversed(tape["ups"]):
            bn, conv = u["bn"], u["conv"]
            g_raw, dgamma, dbeta, _ = dense_train.bn_backward(g, u["raw"], u["st"], bn.weight, None)
            grads[bn.weight], grads[bn.bias] = dgamma, dbeta
            g_low = dense_train.upsample2x_backward(g_raw)
            g_op = dense_train.operand(g_low, mode)
            grads[conv.weight] = dense_train.conv_wgrad(u["inp"], g_op, 1, 1, 1, **dense_train.amp_kw(mode))
            skip_grads.append(g)                                             # + skip: identity
            g = dense_train.conv_dgrad(g_op, conv.weight, 1, *u["inp"].shape[1:3], **dense_train.amp_kw(mode))
        # skip_grads: up1 (skip = the decoder input), up2 (skip = out of layer1), up3 (skip = out of layer2)
        g_x = skip_grads[0]
        stage_skip = {"layer3": skip_grads[2], "layer2": skip_grads[1]}
        blocks = tape["blocks"]
        for i in range(len(blocks) - 1, -1, -1):
            name, r1, r2, rd = blocks[i]
            gy1, gm = self._cbn_backward(r2, g, grads, want_masked=True)
            gx, _ = self._cbn_backward(r1, gy1, grads)
            if rd is not None:
                gd, _ = self._cbn_backward(rd, gm, grads)
                gx += gd
            else:
                gx += gm
            g = gx
            if i > 0 and blocks[i - 1][0] != name:                          # first block of a stage: its input is the
                g += stage_skip[name]                                        # previous stage's output = a skip
        g_first, _ = self._cbn_backward(tape["first"], g, grads, need_input=need_x)
        if not need_x:
            return None, grads
        g_x = g_x + g_first
        return g_x.view(B, S, H, W, C).permute(0, 1, 4, 2, 3).contiguous(), grads


class _DecoderTrainFn(torch.autograd.Function):
    """The whole train-mode decoder as one autograd node: forward keeps the activations and per-channel statistics,
    backward walks the layers in reverse on the train-mode kernels (stp3_b200/dense_train.py).  The backward is not
    itself differentiable (create_graph=True yields an error on use), runs once per forward (retain_graph is refused),
    and refuses weights modified in place between forward and backward."""

    @staticmethod
    def forward(ctx, dec, x, *params):
        outs, tape = dec._train_forward(x)
        ctx.dec, ctx.tape, ctx.params = dec, tape, params
        ctx.versions = [p._version for p in params]
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads_out):
        if ctx.tape is None:
            raise RuntimeError("Decoder (train mode): backward ran a second time through the same forward; the "
                               "activations are released after the first backward (retain_graph is not supported) -- "
                               "run the forward again")
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("Decoder (train mode): a decoder parameter was modified in place between forward and "
                               "backward (e.g. optimizer.step() before loss.backward())")
        tape, ctx.tape = ctx.tape, None
        gx, grads = ctx.dec._train_backward(tape, grads_out, ctx.needs_input_grad[1])
        return (None, gx) + tuple(grads.get(p) for p in ctx.params)
