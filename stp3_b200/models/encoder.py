"""Image encoder with the reference's surface (stp3/models/encoder.py:9-108): a truncated EfficientNet trunk and two
heads (context features, depth logits) at 1/8 resolution.

The trunk is third-party (efficientnet-pytorch 0.7.0, not vendored by the reference and absent from this image;
SURVEY.md §8c): it is taken from `efficientnet_pytorch` when importable, or injected (`backbone=`: any module that
maps (M,3,H,W) -> (reduction_3 (M,c3,H/8,W/8), reduction_4 (M,c4,H/16,W/16))).  The heads -- DeepLabHead +
UpsamplingConcat, the layers this repository owns -- run on the wgmma kernels."""
import math

import torch
import torch.nn as nn

from .. import dense
from ..layers.convolutions import DeepLabHead, UpsamplingConcat


class Encoder(nn.Module):
    REDUCTION = {'b4': [0, 24, 32, 56, 160, 448], 'b0': [0, 16, 24, 40, 112, 320]}

    def __init__(self, cfg, D, backbone=None):
        super().__init__()
        self.D = D
        self.C = cfg.OUT_CHANNELS
        self.use_depth_distribution = cfg.USE_DEPTH_DISTRIBUTION
        self.downsample = cfg.DOWNSAMPLE
        self.version = cfg.NAME.split('-')[1]
        if self.version not in self.REDUCTION:
            raise NotImplementedError
        self.reduction_channel = self.REDUCTION[self.version]
        if backbone is None:
            try:
                from efficientnet_pytorch import EfficientNet
            except ImportError as e:
                raise RuntimeError("efficientnet_pytorch is not installed: pass backbone=<module returning "
                                   "(reduction_3, reduction_4)> to Encoder / STP3") from e
            backbone = EfficientNet.from_pretrained(cfg.NAME)
        if hasattr(backbone, "_conv_stem"):        # an efficientnet_pytorch model: truncate it like encoder.py:39-55
            _truncate_efficientnet(backbone, self.version, self.downsample)
        self.backbone = backbone
        index = int(math.log2(self.downsample))
        c_hi, c_lo = self.reduction_channel[index + 1], self.reduction_channel[index]
        if self.use_depth_distribution:
            self.depth_layer_1 = DeepLabHead(c_hi, c_hi, hidden_channel=64)
            self.depth_layer_2 = UpsamplingConcat(c_hi + c_lo, self.D)
        self.feature_layer_1 = DeepLabHead(c_hi, c_hi, hidden_channel=64)
        self.feature_layer_2 = UpsamplingConcat(c_hi + c_lo, self.C)

    def heads_hl(self, r_lo: torch.Tensor, r_hi: torch.Tensor):
        """r_lo (M,c3,H/8,W/8), r_hi (M,c4,H/16,W/16) fp32 -> (feature HL, depth-logit HL or None)."""
        x = dense.from_f32(r_hi.unsqueeze(1))
        feat = self.feature_layer_2.forward_hl(self.feature_layer_1.forward_hl(x), r_lo)
        depth = None
        if self.use_depth_distribution:
            depth = self.depth_layer_2.forward_hl(self.depth_layer_1.forward_hl(x), r_lo)
        return feat, depth

    def heads_f32(self, r_lo: torch.Tensor, r_hi: torch.Tensor, channels_last: bool = False):
        """Both heads with fp32 outputs written straight from the last convolution's epilogue: context features
        (M,C,Hf,Wf) -- or channels-last (M,Hf,Wf,C), the layout the lift-splat kernel stages with one TMA box per tile
        (SURVEY.md row f1) -- and depth logits (M,D,Hf,Wf) (the reference's layout: they are also a model output)."""
        M, _, Hf, Wf = r_lo.shape
        dev = r_lo.device
        x = dense.from_f32(r_hi.unsqueeze(1))
        feat = torch.empty((M, Hf, Wf, self.C) if channels_last else (M, self.C, Hf, Wf), dtype=torch.float32, device=dev)
        self.feature_layer_2.forward_hl(self.feature_layer_1.forward_hl(x), r_lo, out_f32=feat, out_f32_nhwc=channels_last)
        depth = None
        if self.use_depth_distribution:
            depth = torch.empty((M, self.D, Hf, Wf), dtype=torch.float32, device=dev)
            self.depth_layer_2.forward_hl(self.depth_layer_1.forward_hl(x), r_lo, out_f32=depth)
        return feat, depth

    def trunk(self, x):
        """(M,3,H,W) images -> (reduction_3 (M,c3,H/8,W/8), reduction_4 (M,c4,H/16,W/16)) (encoder.py:57-86)."""
        if hasattr(self.backbone, "_conv_stem"):
            return _efficientnet_endpoints(self.backbone, x)
        return self.backbone(x)

    def get_features_depth(self, x, channels_last: bool = False):
        r_lo, r_hi = self.trunk(x)
        return self.heads_f32(r_lo.float().contiguous(), r_hi.float().contiguous(), channels_last)

    def forward(self, x):
        return self.get_features_depth(x)


def _truncate_efficientnet(net, version, downsample):
    """Drop the blocks and head the ds=8 encoder never uses (keeps the reference's `backbone.*` state-dict keys)."""
    assert downsample == 8
    last = {'b0': 10, 'b4': 21}[version]
    del net._blocks[last + 1:]
    for name in ('_conv_head', '_bn1', '_avg_pooling', '_dropout', '_fc'):
        if hasattr(net, name):
            delattr(net, name)


def _efficientnet_endpoints(net, x):
    """Stem + remaining blocks; returns the 1/8 and 1/16 resolution endpoints (encoder.py:57-86)."""
    x = net._swish(net._bn0(net._conv_stem(x)))
    ends, prev = [], x
    for idx, block in enumerate(net._blocks):
        rate = net._global_params.drop_connect_rate
        if rate:
            rate *= float(idx) / len(net._blocks)
        x = block(x, drop_connect_rate=rate)
        if prev.size(2) > x.size(2):
            ends.append(prev)
        prev = x
    ends.append(x)
    return ends[2], ends[3]
