"""TEST INFRASTRUCTURE -- the train-mode EfficientNet trunk restated in torch autograd (fp64 or fp32), as the reference's
Encoder.get_features_depth drives efficientnet-pytorch 0.7.0 in train mode (stp3/models/encoder.py:57-86): batch-statistics
BatchNorm with running-statistic updates, and drop-connect on the identity-skip blocks with a pinned per-image mask
(out = inputs + x / keep * mask, keep = 1 - 0.2 * idx / len(blocks)).  It walks oracle/efficientnet_oracle.py's modules
(so their parameters get the gradients) and leaves that module's own eval-mode forward untouched."""
import torch
import torch.nn.functional as F

from oracle import efficientnet_oracle as EO


def drop_rates(n_blocks):
    return [0.2 * i / n_blocks for i in range(n_blocks)]


def is_skip(r) -> bool:
    return r['s'] == 1 and r['cin'] == r['cout']


def draw_masks(net, M, device, dtype=torch.float32):
    """The masks the package draws (one torch.rand of M values per skip block with a nonzero rate, in block order):
    {block index: floor(keep + U)} -- seed torch's generator as before the forward being reproduced."""
    n = len(net._blocks)
    masks = {}
    for i, (blk, rate) in enumerate(zip(net._blocks, drop_rates(n))):
        if is_skip(blk.r) and rate > 0:
            masks[i] = torch.floor((1.0 - rate) + torch.rand(M, dtype=dtype, device=device))
    return masks


def block_forward(blk, inputs, rate, mask):
    """MBConvBlock.forward with drop-connect applied through `mask` (M,) on identity-skip blocks."""
    x = inputs
    if blk.r['exp'] != blk.r['cin']:
        x = blk._swish(blk._bn0(blk._expand_conv(inputs)))
    x = blk._swish(blk._bn1(blk._depthwise_conv(x)))
    s = F.adaptive_avg_pool2d(x, 1)
    s = blk._se_expand(blk._swish(blk._se_reduce(s)))
    x = torch.sigmoid(s) * x
    x = blk._bn2(blk._project_conv(x))
    if is_skip(blk.r):
        if mask is not None and rate > 0:
            keep = 1.0 - rate
            x = x / keep * mask.to(x.dtype).view(-1, 1, 1, 1)
        x = x + inputs
    return x


def endpoint_index(net) -> int:
    return max(i for i, b in enumerate(net._blocks) if b.r['s'] == 2) - 1


def trunk_forward(net, x, masks=None):
    """(reduction_3, reduction_4) of the truncated trunk `net` (EO.truncate(EO.EfficientNetOracle(v), v)) on images x,
    in whatever mode net is in; masks: {block index: (M,) keep mask} from draw_masks (None: no drop-connect)."""
    masks = masks or {}
    x = net._swish(net._bn0(net._conv_stem(x)))
    n = len(net._blocks)
    rates = drop_rates(n)
    end = endpoint_index(net)
    r3 = None
    for i, blk in enumerate(net._blocks):
        x = block_forward(blk, x, rates[i], masks.get(i))
        if i == end:
            r3 = x
    return r3, x


def tape_elements(net, H, W) -> int:
    """fp32 elements per image that the native train path keeps (EfficientNetTrunk's tape), counted from the oracle's
    layer shapes: stem output twice; per block the expand output twice, the depthwise output three times (raw, activated,
    gated) and the projection output twice (raw, block output)."""
    sizes = {}
    hooks = []
    for name, m in net.named_modules():
        if isinstance(m, torch.nn.Conv2d) and not name.endswith(('_se_reduce', '_se_expand')):
            hooks.append(m.register_forward_hook(lambda mod, i, o, name=name: sizes.__setitem__(name, o[0].numel())))
    with torch.no_grad():
        net.eval()
        trunk_forward(net, torch.zeros(1, 3, H, W, dtype=next(net.parameters()).dtype))
    for h in hooks:
        h.remove()
    n = 0
    for name, e in sizes.items():
        mult = 3 if name.endswith('_depthwise_conv') else 2
        n += mult * e
    return n



# ------------------------------------------------------------------------------------------------ reduction partitions
# The trunk's partitioned reductions (csrc/trunk_train.cu): the stem and depthwise weight gradients and
# stp3_image_channel_dot split their rows into parts of ceil(rows / parts) consecutive rows, one CTA (row of CTAs) per
# part, and add the parts' fp64 partials in part order.  parts = ceil(rows / rows_per_part), at least 1 and at most
# TR_MAX_PARTS; at the cap the parts grow past rows_per_part, and trailing parts may be empty.
TR_MAX_PARTS = 256


def tr_parts(rows: int, rows_per_part: int) -> int:
    return min(max(-(-rows // rows_per_part), 1), TR_MAX_PARTS)


def stem_wgrad_parts(n_img: int, Ho: int, Wo: int) -> int:
    """parts of stp3_effnet_stem_wgrad over its n_img * Ho * Wo output pixels"""
    return tr_parts(n_img * Ho * Wo, 1024)


def dw_wgrad_parts(n_img: int, Ho: int, Wo: int) -> int:
    """parts of stp3_dw_wgrad over its n_img * Ho * Wo output pixels"""
    return tr_parts(n_img * Ho * Wo, 512)


def dot_parts(hw: int) -> int:
    """parts of stp3_image_channel_dot over the hw pixels of each image"""
    return tr_parts(hw, 256)


def part_features(name: str, rows: int, parts: int, rows_per_part: int) -> set:
    """the partition features of one launch: one part, several parts, a ragged last part (the last non-empty part
    shorter than the others), the part cap (more than TR_MAX_PARTS * rows_per_part rows)"""
    per = -(-rows // parts)
    f = {f"{name} one part" if parts == 1 else f"{name} several parts"}
    if parts > 1 and rows % per:
        f.add(f"{name} ragged last part")
    if rows > TR_MAX_PARTS * rows_per_part:
        f.add(f"{name} part cap")
    return f
