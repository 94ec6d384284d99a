"""ORACLE (test infrastructure) -- train-mode restatement of the TemporalBlocks and TemporalModel
(stp3/layers/temporal.py:252-489 and stp3/models/temporal_model.py:50-60 with every BatchNorm in train mode) in plain
PyTorch, next to oracle/torch_deeplab_train.deeplab_head_train (the head, reused here) and the BatchNorm of
oracle/torch_dense_train.

The parameters are used as they are (no dtype cast), so on a float64 copy of a model (copy.deepcopy(tm).double())
autograd through temporal_model_train is the fp64 gradient oracle.  It never reads the reference.
"""
import torch
import torch.nn.functional as F

from oracle.torch_dense_train import _bn
from oracle.torch_deeplab_train import deeplab_head_train


def temporal_block_train(x, blk, relu=F.relu):
    """x (B, C, T, H, W) -> TemporalBlock.forward in train mode; updates the block's BatchNorm running statistics.
    relu: called in forward order (entry and causal convolution of path 0, the same of path 1, path 2, the pooling
    branch on its T + 1 frames, the aggregation)."""
    paths = []
    for i, path in enumerate(blk.convolution_paths):
        e = path[0] if i < 2 else path
        y = relu(_bn(F.conv3d(x, e.conv.weight), e.norm))
        if i < 2:
            cc = path[1]
            kt, kh, kw = cc.conv.kernel_size
            y = F.pad(y, ((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0))
            y = relu(_bn(F.conv3d(y, cc.conv.weight), cc.norm))
        paths.append(y)
    r = torch.cat(paths, 1)
    if blk.use_pyramid_pooling:
        _, _, _, h, w = x.shape
        pcbr = blk.pyramid_pooling.features[0].conv_bn_relu
        # the reference drops the last pooled frame after the branch's BatchNorm: its statistics cover B*(T+1) values
        m = F.avg_pool3d(x, (2, h, w), stride=(1, h, w), padding=(1, 0, 0), count_include_pad=False)
        v = relu(_bn(F.conv3d(m, pcbr.conv.weight), pcbr.norm))[:, :, :-1]
        r = torch.cat([r, v.expand(-1, -1, -1, h, w)], 1)      # bilinear from a 1x1 map is a broadcast
    agg = blk.aggregation[0]
    r = relu(_bn(F.conv3d(r, agg.conv.weight), agg.norm))
    if blk.projection is not None:
        x = _bn(F.conv3d(x, blk.projection[0].weight), blk.projection[1])
    return x + r


def temporal_model_train(x, tm, relu=F.relu, dropout_mask=None):
    """x (B, S, C, H, W) (every input channel, the ego-motion ones broadcast) -> TemporalModel.forward in train mode
    (B, S, Cout, H, W): the blocks, then the head (oracle.torch_deeplab_train.deeplab_head_train with the same relu
    and dropout_mask)."""
    B, S = x.shape[:2]
    y = x.permute(0, 2, 1, 3, 4)
    for blk in tm.model:
        y = temporal_block_train(y, blk, relu)
    y = y.permute(0, 2, 1, 3, 4).reshape(B * S, -1, *y.shape[-2:])
    y = deeplab_head_train(y, tm.final_conv, relu, dropout_mask)
    return y.view(B, S, *y.shape[1:])


def pair_mean(m, T):
    """The T + 1 pooled frames of per-frame means m (B*T, C) (stp3_temporal_pair_mean): frame t is m[0] at t = 0,
    (m[t-1] + m[t]) / 2 for t < T and m[T-1] at t = T, within each sample -> (B*(T+1), C)."""
    mt = m.view(-1, T, m.shape[-1])
    out = torch.cat([mt[:, :1], 0.5 * (mt[:, :-1] + mt[:, 1:]), mt[:, -1:]], 1)
    return out.reshape(-1, m.shape[-1])
