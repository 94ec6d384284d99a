"""ORACLE (test infrastructure) -- train-mode restatement of UpsamplingConcat (stp3/layers/convolutions.py:183-201 with
both BatchNorms in train mode) and of one encoder head, DeepLabHead -> UpsamplingConcat (stp3/models/encoder.py:88-95), in
plain PyTorch, next to oracle/torch_deeplab_train.deeplab_head_train, whose BatchNorm and dropout handling it shares.

The parameters are used as they are (no dtype cast), so on float64 copies of the modules autograd through these functions
is the fp64 gradient oracle.  It never reads the reference; oracle/make_golden_encoder_train.py pins it to the reference's
own modules (tests/golden/encoder_heads_train.npz).
"""
import torch
import torch.nn.functional as F

from oracle.torch_deeplab_train import deeplab_head_train
from oracle.torch_dense_train import _bn


def upsampling_concat_train(x_to_upsample, x, mod, relu=F.relu):
    """x_to_upsample (N,Cc,h,w), x (N,Cf,2h,2w) -> UpsamplingConcat.forward in train mode; updates the module's BatchNorm
    running statistics.  relu: called in forward order (after the first BatchNorm, after the second); a test can pass one
    that applies given masks, which pins every ReLU branch."""
    y = F.interpolate(x_to_upsample, scale_factor=2, mode='bilinear', align_corners=False)
    y = torch.cat([x, y], dim=1)
    y = relu(_bn(F.conv2d(y, mod.conv[0].weight, padding=1), mod.conv[1]))
    return relu(_bn(F.conv2d(y, mod.conv[3].weight, padding=1), mod.conv[4]))


def encoder_head_train(r_lo, r_hi, layer_1, layer_2, relu=F.relu, dropout_mask=None):
    """One encoder head in train mode: layer_2(layer_1(r_hi), r_lo) with layer_1 a DeepLabHead and layer_2 an
    UpsamplingConcat.  relu is called 7 times by the DeepLab head (see deeplab_head_train), then twice here;
    dropout_mask is the DeepLab head's."""
    return upsampling_concat_train(deeplab_head_train(r_hi, layer_1, relu=relu, dropout_mask=dropout_mask), r_lo,
                                   layer_2, relu=relu)
