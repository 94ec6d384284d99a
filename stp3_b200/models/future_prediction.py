"""FuturePrediction (stp3/models/future_prediction.py), eval mode: Dual_GRU -> ConvNeXt Block per future frame, then
n_gru_blocks SpatialGRUs over the present and future frames, each followed by Blocks (the last by a DeepLabHead).
Both SpatialGRUs start from the first present state, as in the reference."""
import torch
import torch.nn as nn

from .. import dense
from ..layers.convolutions import PREDICT_EVAL_ONLY, Block, DeepLabHead
from ..layers.temporal import Dual_GRU, SpatialGRU


class FuturePrediction(nn.Module):
    def __init__(self, in_channels, latent_dim, n_future, mixture=True, n_gru_blocks=2, n_res_layers=1):
        super(FuturePrediction, self).__init__()
        self.n_spatial_gru = n_gru_blocks
        self.n_future = n_future
        self.in_channels = in_channels
        gru_in_channels = latent_dim
        self.dual_grus = Dual_GRU(gru_in_channels, in_channels, n_future=n_future, mixture=mixture)
        self.res_blocks1 = nn.Sequential(*[Block(in_channels) for _ in range(n_res_layers)])
        self.spatial_grus = []
        self.res_blocks = []
        for i in range(self.n_spatial_gru):
            self.spatial_grus.append(SpatialGRU(in_channels, in_channels))
            if i < self.n_spatial_gru - 1:
                self.res_blocks.append(nn.Sequential(*[Block(in_channels) for _ in range(n_res_layers)]))
            else:
                self.res_blocks.append(DeepLabHead(in_channels, in_channels, 128))
        self.spatial_grus = torch.nn.ModuleList(self.spatial_grus)
        self.res_blocks = torch.nn.ModuleList(self.res_blocks)

    @staticmethod
    def _blocks(seq, x: dense.HL) -> dense.HL:
        if isinstance(seq, DeepLabHead):
            return seq.forward_hl(x)
        for blk in seq:
            x = blk.forward_hl(x)
        return x

    def forward_hl(self, x, state: dense.HL) -> dense.HL:
        """x: HL (B, 1, H, W, >= latent_dim) the latent sample or None (zeros); state: HL (B, S, H, W, 64) the present
        states -> HL (B, S + n_future, H, W, 64)."""
        if any(m.training for m in self.modules()):
            raise NotImplementedError(f"FuturePrediction: {PREDICT_EVAL_ONLY}")
        B, S, H, W, _ = state.hi.shape
        fut = dense.HL.empty(B, self.n_future, H, W, self.in_channels, state.hi.device)
        self.dual_grus.forward_hl(x, state, fut)
        fut = self._blocks(self.res_blocks1, fut)
        frames = [(state, t) for t in range(S)] + [(fut, t) for t in range(self.n_future)]
        h0 = (state, 0)                                # x[:, 0] of cat([state, future]), taken once
        y = None
        for i in range(self.n_spatial_gru):
            y = self.spatial_grus[i].forward_hl(frames, h0)
            y = self._blocks(self.res_blocks[i], y)
            frames = [(y, t) for t in range(S + self.n_future)]
        return y

    def forward(self, x, state):
        """x (B, 1, latent_dim, H, W) fp32, state (B, S, C, H, W) fp32 -> (B, S + n_future, C, H, W) fp32."""
        y = self.forward_hl(dense.from_f32(x) if x is not None else None, dense.from_f32(state))
        return dense.to_f32(y, 0, self.in_channels)
