"""ORACLE (test infrastructure) — plain-PyTorch functional restatement of the dense layers of the hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` leg may import this.

Every function takes a module that carries the REFERENCE'S PARAMETER TREE (either the reference's own module,
imported through oracle/ref_loader.py in the build container, or the drop-in module of stp3_b200, which keeps the
same names) and evaluates the reference semantics with torch.nn.functional ops in the dtype of the input (fp32 like
the reference, or fp64 for a tighter oracle).  Nothing here calls the modules' own forward().

  conv_1x1x1_norm_activated / CausalConv3d   stp3/layers/temporal.py:252-273, 315-325
  PyramidSpatioTemporalPooling               stp3/layers/temporal.py:375-423
  TemporalBlock                              stp3/layers/temporal.py:426-489
  ASPP / DeepLabHead / UpsamplingAdd         stp3/layers/convolutions.py:204-280
  TemporalModel                              stp3/models/temporal_model.py:50-60
  Decoder (+ torchvision BasicBlock)         stp3/models/decoder.py:91-140

Pinned by tests/test_dense_oracle.py: (a) in the build container against the reference modules' own forward on the
same weights, (b) everywhere against tests/golden/dense_*.npz produced from the reference by oracle/make_golden.py.
"""
import torch
import torch.nn.functional as F


# seeded, machine-independent synthetic weights / inputs live with the other synthetic-data helpers
from stp3_b200.utils.synthetic import exact_gauss, init_exact  # noqa: E402,F401


# ------------------------------------------------------------------------------------------------ primitives
def _bn(x, bn):
    shape = [1, -1] + [1] * (x.dim() - 2)
    d = x.dtype
    s = bn.weight.to(d) / torch.sqrt(bn.running_var.to(d) + bn.eps)
    return (x - bn.running_mean.to(d).view(shape)) * s.view(shape) + bn.bias.to(d).view(shape)


def _cna3(x, seq):          # conv_1x1x1_norm_activated
    return F.relu(_bn(F.conv3d(x, seq.conv.weight.to(x.dtype)), seq.norm))


def _causal(x, m):          # CausalConv3d: pad (w, w, h, h, kt-1, 0) then conv/bn/relu
    kt, kh, kw = m.conv.kernel_size
    x = F.pad(x, ((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0))
    return F.relu(_bn(F.conv3d(x, m.conv.weight.to(x.dtype)), m.norm))


def pyramid_pooling(x, pp):
    b, _, t, h, w = x.shape
    outs = []
    for f in pp.features:
        ks = f.avgpool.kernel_size
        y = F.avg_pool3d(x, ks, stride=(1, *ks[1:]), padding=(ks[0] - 1, 0, 0), count_include_pad=False)[:, :, :-1]
        y = _cna3(y.contiguous(), f.conv_bn_relu)
        c = y.shape[1]
        y = F.interpolate(y.permute(0, 2, 1, 3, 4).reshape(b * t, c, *y.shape[-2:]), (h, w), mode='bilinear',
                          align_corners=False)
        outs.append(y.view(b, t, c, h, w).permute(0, 2, 1, 3, 4))
    return torch.cat(outs, 1)


def temporal_block(x, blk):
    """x (B,C,T,H,W)."""
    paths = [_causal(_cna3(x, blk.convolution_paths[0][0]), blk.convolution_paths[0][1]),
             _causal(_cna3(x, blk.convolution_paths[1][0]), blk.convolution_paths[1][1]),
             _cna3(x, blk.convolution_paths[2])]
    r = torch.cat(paths, 1)
    if blk.use_pyramid_pooling:
        r = torch.cat([r, pyramid_pooling(x, blk.pyramid_pooling)], 1)
    r = _cna3(r, blk.aggregation[0])
    if blk.projection is not None:
        x = _bn(F.conv3d(x, blk.projection[0].weight.to(x.dtype)), blk.projection[1])
    return x + r


def deeplab_head(x, head):
    """x (N,C,H,W); head = Sequential(ASPP, conv3x3, bn, relu, conv1x1+bias)."""
    aspp = head[0]
    d = x.dtype
    outs = []
    for br in aspp.convs:
        first = br[0]
        if isinstance(first, torch.nn.AdaptiveAvgPool2d):
            y = x.mean(dim=(2, 3), keepdim=True)
            y = F.relu(_bn(F.conv2d(y, br[1].weight.to(d)), br[2]))
            y = F.interpolate(y, size=x.shape[-2:], mode='bilinear', align_corners=False)
        else:
            y = F.relu(_bn(F.conv2d(x, first.weight.to(d), padding=first.padding, dilation=first.dilation), br[1]))
        outs.append(y)
    y = F.relu(_bn(F.conv2d(torch.cat(outs, 1), aspp.project[0].weight.to(d)), aspp.project[1]))
    y = F.relu(_bn(F.conv2d(y, head[1].weight.to(d), padding=1), head[2]))
    return F.conv2d(y, head[4].weight.to(d), head[4].bias.to(d))


def temporal_model(x, tm):
    """x (B,S,C,H,W) -> (B,S,Cout,H,W)."""
    y = x.permute(0, 2, 1, 3, 4)
    for blk in tm.model:
        y = temporal_block(y, blk)
    y = y.permute(0, 2, 1, 3, 4).contiguous()
    b, s, c, h, w = y.shape
    return deeplab_head(y.view(b * s, c, h, w), tm.final_conv).view(b, s, -1, h, w)


def _basic_block(x, blk):
    d = x.dtype
    y = F.relu(_bn(F.conv2d(x, blk.conv1.weight.to(d), stride=blk.conv1.stride, padding=1), blk.bn1))
    y = _bn(F.conv2d(y, blk.conv2.weight.to(d), padding=1), blk.bn2)
    if blk.downsample is not None:
        x = _bn(F.conv2d(x, blk.downsample[0].weight.to(d), stride=blk.downsample[0].stride), blk.downsample[1])
    return F.relu(y + x)


def upsampling_add(x, skip, up):
    y = F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)
    y = _bn(F.conv2d(y, up.upsample_layer[1].weight.to(x.dtype)), up.upsample_layer[2])
    return y + skip


def _head(x, h):
    d = x.dtype
    y = F.relu(_bn(F.conv2d(x, h[0].weight.to(d), padding=1), h[1]))
    y = F.conv2d(y, h[3].weight.to(d), h[3].bias.to(d))
    return torch.sigmoid(y) if len(h) > 4 else y


def decoder(x, dec):
    """x (B,S,C,H,W) -> dict like Decoder.forward."""
    b, s, c, h, w = x.shape
    d = x.dtype
    x = x.reshape(b * s, c, h, w)
    skip1 = x
    y = F.relu(_bn(F.conv2d(x, dec.first_conv.weight.to(d), stride=2, padding=3), dec.bn1))
    for blk in dec.layer1:
        y = _basic_block(y, blk)
    skip2 = y
    for blk in dec.layer2:
        y = _basic_block(y, blk)
    skip3 = y
    for blk in dec.layer3:
        y = _basic_block(y, blk)
    y = upsampling_add(y, skip3, dec.up3_skip)
    y = upsampling_add(y, skip2, dec.up2_skip)
    y = upsampling_add(y, skip1, dec.up1_skip)
    out = {}
    def per_frame(t):
        return t.view(b, s, *t.shape[1:])
    out['segmentation'] = per_frame(_head(y, dec.segmentation_head))
    out['pedestrian'] = per_frame(_head(y, dec.pedestrian_head)) if dec.predict_pedestrian else None
    out['hdmap'] = _head(y.view(b, s, *y.shape[1:])[:, dec.n_present - 1], dec.hdmap_head) if dec.perceive_hdmap else None
    out['instance_center'] = per_frame(_head(y, dec.instance_center_head)) if dec.predict_instance else None
    out['instance_offset'] = per_frame(_head(y, dec.instance_offset_head)) if dec.predict_instance else None
    out['instance_flow'] = per_frame(_head(y, dec.instance_future_head)) if dec.predict_future_flow else None
    out['costvolume'] = per_frame(_head(y, dec.costvolume_head).squeeze(1)) if dec.planning else None
    return out


def upsampling_concat(x_to_upsample, x, m):
    """UpsamplingConcat (convolutions.py:183-201): upsample the coarse map x2, concat BEHIND the fine map, 2x conv."""
    d = x.dtype
    y = F.interpolate(x_to_upsample, scale_factor=2, mode='bilinear', align_corners=False)
    y = torch.cat([x, y], dim=1)
    y = F.relu(_bn(F.conv2d(y, m.conv[0].weight.to(d), padding=1), m.conv[1]))
    return F.relu(_bn(F.conv2d(y, m.conv[3].weight.to(d), padding=1), m.conv[4]))


def encoder_heads(r_lo, r_hi, enc):
    """Encoder.get_features_depth after the trunk (encoder.py:88-95): r_lo (M,c3,H/8,W/8), r_hi (M,c4,H/16,W/16)."""
    feat = upsampling_concat(deeplab_head(r_hi, enc.feature_layer_1), r_lo, enc.feature_layer_2)
    depth = None
    if enc.use_depth_distribution:
        depth = upsampling_concat(deeplab_head(r_hi, enc.depth_layer_1), r_lo, enc.depth_layer_2)
    return feat, depth
