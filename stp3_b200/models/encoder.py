"""Image encoder with the reference's surface (stp3/models/encoder.py:9-108): a truncated EfficientNet trunk and two
heads (context features, depth logits) at 1/8 resolution.

The trunk (efficientnet-pytorch 0.7.0, not vendored by the reference; SURVEY.md §8c) is chosen by `backbone=`:
  "native"      the sm_90a trunk of this package (models/efficientnet.py, same state-dict keys);
  None          efficientnet_pytorch's pretrained model when the package is importable, else the native trunk;
  a module      injected: maps (M,3,H,W) -> (reduction_3 (M,c3,H/8,W/8), reduction_4 (M,c4,H/16,W/16)).
The heads -- DeepLabHead + UpsamplingConcat -- run on the wgmma kernels.  With the native trunk the endpoints reach the
heads as hi/lo planes: block 9 writes reduction_3 straight into the heads' concat tensor.

The heads also run in train mode (batch statistics, dropout, autograd; DeepLabHead.forward and
UpsamplingConcat.forward on fp32 endpoints).  The default native trunk is eval-only: with it the endpoints are computed
under no_grad and train_heads() gives the frozen-trunk fine-tune.  A native trunk built with
EfficientNetTrunk(version, trainable=True) follows nn.Module.train(): in train mode its endpoints leave the trunk as fp32
tensors with a grad_fn (channels-last memory, NCHW views) and receive the gradients of both heads.  An injected torch
trunk follows nn.Module.train() and receives the gradients of both endpoints through torch autograd."""
import math

import torch
import torch.nn as nn

from .. import dense
from ..layers.convolutions import DeepLabHead, UpsamplingConcat
from .efficientnet import EfficientNetTrunk


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
                backbone = EfficientNet.from_pretrained(cfg.NAME)
            except ImportError:
                backbone = "native"
        if isinstance(backbone, str):
            if backbone != "native":
                raise ValueError(f"backbone={backbone!r}: pass 'native', None or a module")
            backbone = EfficientNetTrunk(self.version, self.downsample)
        if hasattr(backbone, "_conv_stem") and not isinstance(backbone, EfficientNetTrunk):
            # an efficientnet_pytorch model: truncate it like encoder.py:39-55 (the native trunk is built truncated)
            _truncate_efficientnet(backbone, self.version, self.downsample)
        self.backbone = backbone
        index = int(math.log2(self.downsample))
        c_hi, c_lo = self.reduction_channel[index + 1], self.reduction_channel[index]
        if self.use_depth_distribution:
            self.depth_layer_1 = DeepLabHead(c_hi, c_hi, hidden_channel=64)
            self.depth_layer_2 = UpsamplingConcat(c_hi + c_lo, self.D)
        self.feature_layer_1 = DeepLabHead(c_hi, c_hi, hidden_channel=64)
        self.feature_layer_2 = UpsamplingConcat(c_hi + c_lo, self.C)

    def _head_modules(self):
        mods = [self.feature_layer_1, self.feature_layer_2]
        if self.use_depth_distribution:
            mods += [self.depth_layer_1, self.depth_layer_2]
        return mods

    def heads_training(self) -> bool:
        """True when the head modules are in train mode; they must all be in the same mode."""
        modes = {m.training for m in self._head_modules()}
        if len(modes) > 1:
            raise RuntimeError("Encoder: the head modules (feature_layer_1/2, depth_layer_1/2) are in mixed train / eval "
                               "modes; call encoder.train_heads(True) or encoder.train_heads(False)")
        return modes.pop()

    def train_heads(self, mode: bool = True):
        """Sets the four head modules' mode and leaves the trunk alone: model.eval(); model.encoder.train_heads() is the
        frozen-trunk recipe, for the default (eval-only) native trunk and a trainable one alike.  Returns self."""
        for m in self._head_modules():
            m.train(mode)
        return self

    def heads_train(self, r_lo: torch.Tensor, r_hi: torch.Tensor, channels_last: bool = False):
        """heads_f32 with the heads in train mode: outputs carry a grad_fn; both heads read the same endpoints, autograd
        adds their two gradients."""
        feat = self.feature_layer_2(self.feature_layer_1(r_hi), r_lo, channels_last=channels_last)
        depth = self.depth_layer_2(self.depth_layer_1(r_hi), r_lo) if self.use_depth_distribution else None
        return feat, depth

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
        if self.heads_training():
            return self.heads_train(r_lo, r_hi, channels_last)
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

    @property
    def native(self) -> bool:
        return isinstance(self.backbone, EfficientNetTrunk)

    def trunk_training(self) -> bool:
        """True when the native trunk is in train mode (a trunk built with trainable=True, after train())."""
        return self.native and self.backbone.training

    def features_native(self, x: torch.Tensor, channels_last: bool = False):
        """(M,3,H,W) fp32 images -> heads_f32's outputs through the native trunk, hi/lo from the stem to the heads."""
        if self.heads_training():
            if self.trunk_training():
                r_lo, r_hi = self.backbone(x)     # fp32 endpoints with a grad_fn: the trunk trains too
            else:
                with torch.no_grad():             # the native trunk is frozen: fp32 endpoints, no graph behind them
                    r_lo, r_hi = self.backbone(x)
            return self.heads_train(r_lo, r_hi, channels_last)
        if self.trunk_training():
            raise RuntimeError("Encoder: the native trunk is in train mode but the heads are in eval mode, so no "
                               "gradient could reach it -- call encoder.train_heads() as well, or backbone.eval()")
        M, _, H, W = x.shape
        ds = self.downsample
        index = int(math.log2(ds))
        c_hi, c_lo = self.reduction_channel[index + 1], self.reduction_channel[index]
        cat = dense.HL.empty(M, 1, H // ds, W // ds, c_lo + c_hi, x.device)
        r_lo, r_hi = self.backbone.forward_hl(x, r3_out=cat)
        assert r_lo is cat and r_hi.hi.shape[2:4] == (H // (2 * ds), W // (2 * ds)), "image size must be a multiple of 16"
        Hf, Wf = H // ds, W // ds
        feat = torch.empty((M, Hf, Wf, self.C) if channels_last else (M, self.C, Hf, Wf), dtype=torch.float32,
                           device=x.device)
        self.feature_layer_2.forward_cat(self.feature_layer_1.forward_hl(r_hi), cat, c_lo, out_f32=feat,
                                         out_f32_nhwc=channels_last)
        depth = None
        if self.use_depth_distribution:
            depth = torch.empty((M, self.D, Hf, Wf), dtype=torch.float32, device=x.device)
            self.depth_layer_2.forward_cat(self.depth_layer_1.forward_hl(r_hi), cat, c_lo, out_f32=depth)
        return feat, depth

    def trunk(self, x):
        """(M,3,H,W) images -> (reduction_3 (M,c3,H/8,W/8), reduction_4 (M,c4,H/16,W/16)) (encoder.py:57-86)."""
        if self.native:
            return self.backbone(x.float().contiguous())
        if hasattr(self.backbone, "_conv_stem"):
            return _efficientnet_endpoints(self.backbone, x)
        return self.backbone(x)

    def get_features_depth(self, x, channels_last: bool = False):
        if self.native:
            return self.features_native(x.float().contiguous(), channels_last)
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
