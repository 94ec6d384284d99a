"""ORACLE (test infrastructure) -- train-mode restatement of the DeepLab head (stp3/layers/convolutions.py:204-280 with
every BatchNorm in train mode and its Dropout) in plain PyTorch, next to oracle/torch_dense.deeplab_head (the eval-mode
one) and oracle/torch_dense_train.decoder_train (the train-mode decoder, whose BatchNorm it shares).

The parameters are used as they are (no dtype cast), so on a float64 copy of a head (copy.deepcopy(head).double())
autograd through deeplab_head_train is the fp64 gradient oracle.  It never reads the reference;
oracle/make_golden_head_train.py pins it to the reference's own DeepLabHead (tests/golden/deeplab_train_*.npz).
"""
import torch
import torch.nn.functional as F

from oracle.torch_dense_train import _bn


def deeplab_head_train(x, head, relu=F.relu, dropout_mask=None):
    """x (N,C,H,W) -> DeepLabHead.forward in train mode; updates the head's BatchNorm running statistics.
    relu: called in forward order (the four spatial ASPP branches, the pooling branch, the projection, the 3x3);
    dropout_mask: the keep mask of ASPP.project[3] (N, hidden, H, W), scaled by 1 / (1 - p) here, or None for a fresh
    F.dropout draw."""
    aspp = head[0]
    outs = []
    for br in aspp.convs:
        first = br[0]
        if isinstance(first, torch.nn.AdaptiveAvgPool2d):
            y = relu(_bn(F.conv2d(x.mean(dim=(2, 3), keepdim=True), br[1].weight), br[2]))
            y = F.interpolate(y, size=x.shape[-2:], mode='bilinear', align_corners=False)
        else:
            y = relu(_bn(F.conv2d(x, first.weight, padding=first.padding, dilation=first.dilation), br[1]))
        outs.append(y)
    y = relu(_bn(F.conv2d(torch.cat(outs, 1), aspp.project[0].weight), aspp.project[1]))
    p = aspp.project[3].p
    y = F.dropout(y, p, True) if dropout_mask is None else y * dropout_mask.to(y.dtype) * (1.0 / (1.0 - p))
    y = relu(_bn(F.conv2d(y, head[1].weight, padding=1), head[2]))
    return F.conv2d(y, head[4].weight, head[4].bias)


def dropout_keep_mask(shape, seed: int, p: float = 0.5) -> torch.Tensor:
    """A machine-independent Bernoulli(1 - p) keep mask (bool) from the integer mt19937 stream (the stream
    stp3_b200.utils.synthetic draws its fixtures from), for fixtures."""
    u = torch.randint(0, 1 << 24, tuple(shape), generator=torch.Generator().manual_seed(seed), dtype=torch.int64)
    return u >= int(p * (1 << 24))
