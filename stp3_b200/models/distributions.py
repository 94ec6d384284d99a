"""Present distribution of the Prediction configurations (stp3/models/distributions.py), eval mode, GAUSSIAN only:
four downsampling Bottlenecks, global average, 1x1 conv (bias) -> (mu, log sigma).  The mean is the existing spatial
sum (stp3_spatial_sum[_det]) and the 1x1 conv stp3_small_linear with 1 / (H W) folded into its weights."""
import torch
import torch.nn as nn

from .. import dense
from ..layers._packing import PackedModule
from ..layers.convolutions import PREDICT_EVAL_ONLY, Bottleneck


class DistributionModule(PackedModule):
    def __init__(self, in_channels, latent_dim, method="GAUSSIAN"):
        super().__init__()
        if method != 'GAUSSIAN':
            raise NotImplementedError(f"PROBABILISTIC.METHOD = {method}: only the GAUSSIAN present distribution is built "
                                      "on sm_90a (BERNOULLI / MIXGAUSSIAN are not)")
        self.compress_dim = in_channels // 2
        self.latent_dim = latent_dim
        self.method = method
        self.encoder = DistributionEncoder(in_channels, self.compress_dim)
        self.decoder = nn.Sequential(
            nn.AdaptiveAvgPool2d(1), nn.Conv2d(self.compress_dim, out_channels=2 * self.latent_dim, kernel_size=1))

    def _pack(self):
        conv = self.decoder[1]
        return {"w": conv.weight.detach().float().reshape(2 * self.latent_dim, self.compress_dim),
                "b": conv.bias.detach().float().contiguous()}

    def forward_hl(self, s_t: dense.HL) -> torch.Tensor:
        """s_t: HL (B, 1, H, W, >= in_channels) -> (B, 2 * latent_dim) fp32: mu | log sigma."""
        if any(m.training for m in self.modules()):
            raise NotImplementedError(f"DistributionModule: {PREDICT_EVAL_ONLY}")
        P = self.packed()
        y = self.encoder.forward_hl(s_t)
        B, T, h, w, cs = y.hi.shape
        key = ("w_mean", h * w, cs)
        if key not in P:            # the 1x1 conv's weights over the padded sums, times 1 / (h w)
            wm = torch.zeros((2 * self.latent_dim, cs), dtype=torch.float32, device=P["w"].device)
            wm[:, :self.compress_dim] = P["w"] / (h * w)
            P[key] = wm
        out = torch.empty((B * T, 2 * self.latent_dim), dtype=torch.float32, device=y.hi.device)
        dense.small_linear(dense.spatial_sum(y), P[key], out, False, bias=P["b"])
        return out

    def forward(self, s_t):
        """s_t (B, 1, C, H, W) fp32 -> (B, 1, 2 * latent_dim) fp32."""
        b, s = s_t.shape[:2]
        assert s == 1
        return self.forward_hl(dense.from_f32(s_t)).view(b, 1, 2 * self.latent_dim)


class DistributionEncoder(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.model = nn.Sequential(
            Bottleneck(in_channels, out_channels=out_channels, downsample=True),
            Bottleneck(out_channels, out_channels=out_channels, downsample=True),
            Bottleneck(out_channels, out_channels=out_channels, downsample=True),
            Bottleneck(out_channels, out_channels=out_channels, downsample=True),
        )

    def forward_hl(self, s_t: dense.HL) -> dense.HL:
        for m in self.model:
            s_t = m.forward_hl(s_t)
        return s_t
