"""TemporalModel with the reference's constructor/forward surface (stp3/models/temporal_model.py:7-70)."""
import torch
import torch.nn as nn

from .. import dense
from ..layers.convolutions import DeepLabHead
from ..layers.temporal import TemporalBlock


class TemporalModel(nn.Module):
    def __init__(self, in_channels, receptive_field, input_shape, start_out_channels=64, extra_in_channels=0,
                 n_spatial_layers_between_temporal_layers=0, use_pyramid_pooling=True):
        super().__init__()
        if n_spatial_layers_between_temporal_layers != 0:
            raise NotImplementedError("INBETWEEN_LAYERS > 0 (Bottleneck3D) is not used by any reference config")
        self.receptive_field = receptive_field
        h, w = input_shape
        blocks = []
        block_in, block_out = in_channels, start_out_channels
        for _ in range(receptive_field - 1):
            blocks.append(TemporalBlock(block_in, block_out, use_pyramid_pooling=bool(use_pyramid_pooling),
                                        pool_sizes=[(2, h, w)] if use_pyramid_pooling else None))
            block_in = block_out
            block_out += extra_in_channels
        self.out_channels = block_in
        self.final_conv = DeepLabHead(block_out, block_out, hidden_channel=128)
        self.model = nn.Sequential(*blocks)

    def forward_hl(self, x: dense.HL, const=None, sums=None):
        """x: HL (B, S, H, W, .) -> HL with the head's channels; with final_conv in train mode (and the blocks in eval
        mode) an fp32 (B, S, C, H, W) tensor with a grad_fn instead (the head's batch statistics, dropout, autograd)."""
        n_img = x.hi.shape[0] * x.hi.shape[1]
        for i, block in enumerate(self.model):
            # a 64-channel block hands the spatial sums of its output (the next block's pyramid pooling / the head's
            # global-pool branch need them) over from its aggregation conv's epilogue
            nxt = None
            if block.out_channels <= 64:
                nxt = torch.empty((n_img, 64), dtype=torch.float32, device=x.hi.device)
            x = block.forward_hl(x, const if i == 0 else None, sums, out_sums=nxt)
            sums = nxt
        if self.final_conv.training:
            B, S = x.hi.shape[:2]
            y = self.final_conv(dense.to_f32(x, 0, self.final_conv.in_channels).flatten(0, 1))
            return y.view(B, S, *y.shape[1:])
        return self.final_conv.forward_hl(x, sums=sums)

    def forward(self, x):
        """x (B, S, C, H, W) fp32 -> (B, S, Cout, H, W) fp32."""
        y = self.forward_hl(dense.from_f32(x))
        return y if torch.is_tensor(y) else dense.to_f32(y, 0, self.final_conv.num_classes)


class TemporalModelIdentity(nn.Module):
    def __init__(self, in_channels, receptive_field):
        super().__init__()
        self.receptive_field = receptive_field
        self.out_channels = in_channels

    def forward(self, x):
        return x
