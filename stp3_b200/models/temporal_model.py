"""TemporalModel with the reference's constructor/forward surface (stp3/models/temporal_model.py:7-70)."""
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .. import dense, dense_train
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

    def blocks_training(self) -> bool:
        """True when the TemporalBlocks run in train mode.  They train together, and only with the head in train mode
        too: with an eval-mode head no gradient could reach them."""
        modes = {blk.training for blk in self.model}
        if len(modes) > 1:
            raise RuntimeError("TemporalModel: the TemporalBlocks are in mixed train / eval modes; they train together "
                               "(call .train() or .eval() on temporal_model.model as a whole)")
        training = modes == {True}
        if training and not self.final_conv.training:
            raise RuntimeError("TemporalModel: the TemporalBlocks are in train mode but final_conv is in eval mode, so "
                               "no gradient could reach them -- call final_conv.train() as well")
        return training

    def forward_hl(self, x, const=None, sums=None):
        """x: HL (B, S, H, W, .) -> HL with the head's channels; with final_conv in train mode (and the blocks in eval
        mode) an fp32 (B, S, C, H, W) tensor with a grad_fn instead (the head's batch statistics, dropout, autograd).
        With the blocks in train mode too, x may also be an fp32 (B, S, C, H, W) tensor (its gradient is computed when
        it requires grad); const (B*S, n_const) are the spatially constant input channels of the first block."""
        if self.blocks_training():
            return self._forward_train(dense.to_f32(x, 0, x.c) if isinstance(x, dense.HL) else x, const)
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

    def forward(self, x, const=None):
        """x (B, S, C, H, W) fp32 -> (B, S, Cout, H, W) fp32; const (B*S, n_const): the first block's spatially constant
        input channels (the ego-motion under STP3), behind the C channels of x."""
        if self.blocks_training():
            return self._forward_train(x, const)
        y = self.forward_hl(dense.from_f32(x), const=const)
        return y if torch.is_tensor(y) else dense.to_f32(y, 0, self.final_conv.num_classes)

    # ------------------------------------------------------------------------------------------------ train mode
    def _forward_train(self, x: torch.Tensor, const):
        """The blocks and the head in train mode: (B, S, Cout, H, W) fp32 with a grad_fn."""
        for i, blk in enumerate(self.model):
            for name, m in blk.named_modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm):
                    dense_train.check_bn(m, f"TemporalModel.model.{i}.{name}")
        if not x.is_cuda or not self.final_conv[1].weight.is_cuda:
            raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
        B, S = x.shape[:2]
        nc = self.model[0].n_const if len(self.model) else 0
        if (0 if const is None else const.shape[-1]) != nc:
            raise ValueError(f"TemporalModel: the first block takes {nc} spatially constant channels (n_const), got "
                             f"const of shape {None if const is None else tuple(const.shape)}")
        if B * S * dense_train.sync_world(self.final_conv[0].convs[-1][2], B * S, "TemporalModel") < 2:
            # a deliberate refusal of the native path, not the reference's error: the head behind the blocks takes its
            # ASPP pooling statistics over the B*S frames (the process group's under SyncBatchNorm) and would see one
            # value per channel
            raise ValueError("TemporalModel (train mode): B*S = 1 is not supported in train mode (the head's ASPP "
                             "pooling BatchNorm would see one value per channel); train on at least 2 frames")
        const = const.detach().float().reshape(B * S, nc).contiguous() if nc else None
        params = [p for blk in self.model for p in blk.parameters()]
        y = _TemporalBlocksTrainFn.apply(self, x.float(), const, *params) if len(self.model) else x.flatten(0, 1)
        y = self.final_conv(y)
        return y.view(B, S, *y.shape[1:])


class _TemporalBlocksTrainFn(torch.autograd.Function):
    """The train-mode TemporalBlock stack as one autograd node, like the head's (_DeepLabTrainFn): forward keeps the
    activations and statistics of every block, backward walks the blocks in reverse on the train-mode kernels.  x
    (B, S, C, H, W) -> (B*S, Cout, H, W), the head's input.  The backward is not itself differentiable, runs once per
    forward (retain_graph is refused), and refuses weights modified in place between forward and backward."""

    @staticmethod
    def forward(ctx, model, x, const, *params):
        B, S, C, H, W = x.shape
        y = x.detach().permute(0, 1, 3, 4, 2).reshape(B * S, H, W, C).contiguous()
        tapes = []
        for i, blk in enumerate(model.model):
            y, tape = blk._train_forward(y, const if i == 0 else None, B, S)
            tapes.append(tape)
        ctx.model, ctx.tapes, ctx.params, ctx.shape = model, tapes, params, (B, S, C, H, W)
        ctx.versions = [p._version for p in params]
        return y.permute(0, 3, 1, 2).contiguous()

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        if ctx.tapes is None:
            raise RuntimeError("TemporalModel (train mode): backward ran a second time through the same forward; the "
                               "activations are released after the first backward (retain_graph is not supported) -- "
                               "run the forward again")
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("TemporalModel (train mode): a TemporalBlock parameter was modified in place between "
                               "forward and backward (e.g. optimizer.step() before loss.backward())")
        tapes, ctx.tapes = ctx.tapes, None
        B, S, C, H, W = ctx.shape
        g = g_out.float().permute(0, 2, 3, 1).contiguous()
        grads = {}
        blocks = list(ctx.model.model)
        for i in reversed(range(len(blocks))):
            g, gi = blocks[i]._train_backward(tapes[i], g, need_x=i > 0 or ctx.needs_input_grad[1])
            grads.update(gi)
        gx = g.view(B, S, H, W, C).permute(0, 1, 4, 2, 3).contiguous() if g is not None else None
        return (None, gx, None) + tuple(grads.get(p) for p in ctx.params)


class TemporalModelIdentity(nn.Module):
    def __init__(self, in_channels, receptive_field):
        super().__init__()
        self.receptive_field = receptive_field
        self.out_channels = in_channels

    def forward(self, x):
        return x
