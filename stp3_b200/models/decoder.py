"""BEV decoder with the reference's constructor/forward surface and parameter names (stp3/models/decoder.py:8-140):
ResNet-18 stages 1-3 as a U-Net over the BEV grid and 3x3 -> 1x1 heads, executed on the wgmma kernels."""
import torch
import torch.nn as nn
from torchvision.models.resnet import resnet18

from .. import dense
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
        """x (B, S, C, H, W) fp32 -> dict of logits with the reference's keys and shapes (decoder.py:122-140)."""
        return self.forward_hl(dense.from_f32(x))
