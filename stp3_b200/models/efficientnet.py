"""Native EfficientNet trunk (efficientnet-pytorch 0.7.0, b4 and b0) truncated for the ds = 8 encoder like
stp3/models/encoder.py:39-55: the stem and blocks 0..21 (b4) / 0..10 (b0), with the package's attribute names, so a
released ST-P3 checkpoint's `encoder.backbone.*` keys load with strict=True.

Eval mode, per MBConv block (include/stp3_b200.h):
    _expand_conv + _bn0 + swish      stp3_conv_fwd (swish), in column chunks of <= 128 output channels
    _depthwise_conv + _bn1 + swish   stp3_dw_fwd, which also emits the squeeze-excite spatial sums
    squeeze-excite                   stp3_se_gate: the gate of every image folded into per-image projection weights
    _project_conv + _bn2 (+ skip)    stp3_conv_fwd with per-image weights (and res_mode 1 for the identity skip)
BatchNorm eps is each module's own (1e-3 in the trunk).  Activations stay bf16 hi/lo planes from the stem to both
endpoints: reduction_3 (block 9 / 5 output, 1/8) and reduction_4 (block 21 / 10 output, 1/16).

Train mode is opt-in: EfficientNetTrunk(version, trainable=True).train() runs stem -> blocks as one autograd node
(_TrunkTrainFn) on the train-mode kernels with batch-statistics BatchNorm and drop-connect; see _train_forward.  The
default trunk refuses train(): training keeps a large tape (trunk_tape_bytes: 308 MB per 224 x 480 b4 image)."""
import dataclasses
import math
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .. import dense, dense_train
from ..layers._packing import PackedModule

# (width, depth, nominal image size, last block kept for ds = 8) -- efficientnet_pytorch.utils.efficientnet_params
PARAMS = {'b4': (1.4, 1.8, 380, 21), 'b0': (1.0, 1.0, 224, 10)}
# (repeats, kernel, stride, expand ratio, in, out) of the seven stages -- efficientnet_pytorch.utils.efficientnet
STAGES = [(1, 3, 1, 1, 32, 16), (2, 3, 2, 6, 16, 24), (2, 5, 2, 6, 24, 40), (3, 3, 2, 6, 40, 80),
          (3, 5, 1, 6, 80, 112), (4, 5, 2, 6, 112, 192), (1, 3, 1, 6, 192, 320)]
BN_EPS, BN_MOMENTUM = 1e-3, 0.01


def round_filters(f: float, width: float, divisor: int = 8) -> int:
    f *= width
    n = max(divisor, int(f + divisor / 2) // divisor * divisor)
    if n < 0.9 * f:
        n += divisor
    return int(n)


def same_pad(k: int, s: int, size: int) -> Tuple[int, int]:
    """Static 'same' padding (top/left, bottom/right) of a k x k stride-s layer at nominal input size `size`."""
    p = max((math.ceil(size / s) - 1) * s + k - size, 0)
    return p // 2, p - p // 2


@dataclasses.dataclass(frozen=True)
class BlockSpec:
    cin: int
    exp: int
    cout: int
    k: int
    stride: int
    se: int
    pad: Tuple[int, int]

    @property
    def skip(self) -> bool:
        return self.stride == 1 and self.cin == self.cout


def trunk_table(version: str) -> Tuple[int, Tuple[int, int], List[BlockSpec]]:
    """(stem channels, stem pad, block specs) of the truncated trunk."""
    width, depth, size, last = PARAMS[version]
    stem_pad = same_pad(3, 2, size)
    size = math.ceil(size / 2)
    rows = []
    for reps, k, s, e, i, o in STAGES:
        i, o, reps = round_filters(i, width), round_filters(o, width), int(math.ceil(depth * reps))
        for j in range(reps):
            cin, st = (i, s) if j == 0 else (o, 1)
            rows.append(BlockSpec(cin, cin * e, o, k, st, max(1, int(cin * 0.25)), same_pad(k, st, size)))
            if j == 0:
                size = math.ceil(size / s)
    return round_filters(32, width), stem_pad, rows[:last + 1]


def out_size(n: int, k: int, s: int, pad: Tuple[int, int]) -> int:
    return (n + pad[0] + pad[1] - k) // s + 1


def drop_connect_rates(n_blocks: int) -> List[float]:
    """Drop-connect rate of each block of the truncated trunk, 0.2 * idx / len(blocks) (stp3/models/encoder.py:67-69);
    it applies on the identity-skip blocks whose rate is nonzero."""
    return [0.2 * i / n_blocks for i in range(n_blocks)]


def trunk_tape_bytes(version: str, H: int, W: int) -> int:
    """fp32 bytes per image that a train-mode forward keeps for the backward at image size H x W: the stem's raw output
    and activation; per block its input (the previous activation), the expand output before and after _bn0 + swish, the
    depthwise output before and after _bn1 + swish, the gated projection input and the projection output.  Statistics,
    gates and sums are per channel and left out."""
    stem, stem_pad, specs = trunk_table(version)
    h, w = out_size(H, 3, 2, stem_pad), out_size(W, 3, 2, stem_pad)
    n = 2 * stem * h * w
    for s in specs:
        ho, wo = out_size(h, s.k, s.stride, s.pad), out_size(w, s.k, s.stride, s.pad)
        n += (2 * s.exp * h * w if s.exp != s.cin else 0) + 3 * s.exp * ho * wo + 2 * s.cout * ho * wo
        h, w = ho, wo
    return 4 * n


def _bn(c):
    return nn.BatchNorm2d(c, momentum=BN_MOMENTUM, eps=BN_EPS)


class MBConvBlock(nn.Module):
    """Parameter holder with efficientnet-pytorch's names; EfficientNetTrunk runs it."""

    def __init__(self, spec: BlockSpec):
        super().__init__()
        self.spec = spec
        if spec.exp != spec.cin:
            self._expand_conv = nn.Conv2d(spec.cin, spec.exp, 1, bias=False)
            self._bn0 = _bn(spec.exp)
        self._depthwise_conv = nn.Conv2d(spec.exp, spec.exp, spec.k, stride=spec.stride, groups=spec.exp, bias=False)
        self._bn1 = _bn(spec.exp)
        self._se_reduce = nn.Conv2d(spec.exp, spec.se, 1)
        self._se_expand = nn.Conv2d(spec.se, spec.exp, 1)
        self._project_conv = nn.Conv2d(spec.exp, spec.cout, 1, bias=False)
        self._bn2 = _bn(spec.cout)


class EfficientNetTrunk(PackedModule):
    """trainable=False (the default): eval mode only, train() raises.  trainable=True: train() and eval() work like any
    module; eval runs the same folded, packed kernels, train the batch-statistics path of _train_forward.  The state
    dict is the same either way."""

    def __init__(self, version: str = 'b4', downsample: int = 8, trainable: bool = False):
        super().__init__()
        if version not in PARAMS:
            raise NotImplementedError(f"EfficientNet-{version}: the native trunk covers b4 and b0")
        if downsample != 8:
            raise NotImplementedError("the native trunk is truncated for the ds = 8 encoder")
        self.version = version
        self.trainable = bool(trainable)
        stem, self.stem_pad, specs = trunk_table(version)
        self._conv_stem = nn.Conv2d(3, stem, 3, stride=2, bias=False)
        self._bn0 = _bn(stem)
        self._blocks = nn.ModuleList(MBConvBlock(s) for s in specs)
        # reduction_3: the output of the block before the last stride-2 block (the one that leads to 1/16)
        self.endpoint = max(i for i, s in enumerate(specs) if s.stride == 2) - 1
        self.stage_events = None        # tools/trunk_bench.py sets this to a list to receive (stage, CUDA event) marks
        nn.Module.train(self, False)

    def _mark(self, name):
        if self.stage_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))

    def train(self, mode: bool = True):
        if mode and not self.trainable:
            raise NotImplementedError("EfficientNetTrunk: the sm_90a trunk implements the eval-mode forward only "
                                      "(BatchNorm folded into the kernels); training the trunk is not supported. "
                                      "EfficientNetTrunk(version, trainable=True) builds a trunk that trains")
        return nn.Module.train(self, mode)

    # ------------------------------------------------------------------------------------------------ packing
    def _pack(self):
        w, b = dense.fold_bn(self._conv_stem.weight, self._bn0)
        P = {"stem": (w.contiguous(), b.contiguous()), "blocks": []}
        for blk in self._blocks:
            s: BlockSpec = blk.spec
            cpe = dense.pad_to(s.exp)
            B = {}
            if s.exp != s.cin:
                w, b = dense.fold_bn(blk._expand_conv.weight, blk._bn0)
                B["expand"] = [(n0, dense.pack_conv(w[n0:n0 + n].contiguous(), b[n0:n0 + n], bn=bn))
                               for n0, n, bn in dense.se_chunks(s.exp)]
            w, b = dense.fold_bn(blk._depthwise_conv.weight, blk._bn1)          # (exp, 1, k, k)
            dw_w = torch.zeros((s.k * s.k, cpe), dtype=torch.float32, device=w.device)
            dw_w[:, :s.exp] = w.reshape(s.exp, s.k * s.k).t()
            dw_b = torch.zeros(cpe, dtype=torch.float32, device=w.device)
            dw_b[:s.exp] = b
            B["dw"] = (dw_w.contiguous(), dw_b)
            B["se"] = tuple(t.detach().float().reshape(t.shape[0], -1).contiguous() if t.dim() > 1 else
                            t.detach().float().contiguous()
                            for t in (blk._se_reduce.weight, blk._se_reduce.bias, blk._se_expand.weight,
                                      blk._se_expand.bias))
            w, b = dense.fold_bn(blk._project_conv.weight, blk._bn2)
            B["proj_w"] = w.reshape(s.cout, s.exp).contiguous()
            # one PackedConv per column chunk carries the launch geometry and bias; its weights are replaced per call
            # by the chunk's view of the per-image weights stp3_se_gate writes
            proj, off = [], 0
            k_hi = (s.exp + 15) // 16 * 16
            for n0, n, bn in dense.se_chunks(s.cout):
                bias = torch.zeros(bn, dtype=torch.float32, device=w.device)
                bias[:n] = b[n0:n0 + n]
                dense._PACK_COUNTER += 1
                pc = dense.PackedConv(torch.empty(0), bias, [(0, 0, 0)], cpe, bn, n, 1, 0,
                                      k_hi if k_hi > cpe - dense.KB else 0, dense._PACK_COUNTER)
                proj.append((n0, off, pc))
                off += (cpe // dense.KB) * 2 * bn * dense.KB
            B["proj"] = proj
            P["blocks"].append(B)
        return P

    # ------------------------------------------------------------------------------------------------ forward
    def forward_block(self, i: int, x: dense.HL, out: Optional[dense.HL] = None,
                      gate: Optional[torch.Tensor] = None) -> dense.HL:
        """MBConv block i on x (B, T, H, W, .) -> (B, T, Ho, Wo, .) hi/lo; `out` may be a wider tensor (channels
        [0, pad_to(cout)) are written); gate: optional (B*T, exp) fp32 squeeze-excite gate output."""
        s: BlockSpec = self._blocks[i].spec
        B = self.packed()["blocks"][i]
        nb, nt, H, W, _ = x.hi.shape
        dev = x.hi.device
        h = x
        if "expand" in B:
            h = dense.HL.empty(nb, nt, H, W, s.exp, dev)
            for n0, pc in B["expand"]:
                dense.conv(x, pc, out=h, out_coff=n0, swish=True)
            self._mark("expand")
        Ho, Wo = out_size(H, s.k, s.stride, s.pad), out_size(W, s.k, s.stride, s.pad)
        dw_w, dw_b = B["dw"]
        sums = torch.empty((nb * nt, dw_b.numel()), dtype=torch.float32, device=dev)
        # static pads are (before, after) per axis; the kernels take the top / left ones
        y = dense.dw_conv(h, dw_w, dw_b, s.k, s.stride, (s.pad[0], s.pad[0]), (Ho, Wo), sums=sums)
        self._mark("depthwise")
        w_img = dense.se_gate(sums, Ho * Wo, s.exp, *B["se"], B["proj_w"], gate=gate)
        self._mark("se_gate")
        if out is None:
            out = dense.HL.empty(nb, nt, Ho, Wo, s.cout, dev)
        out.c = s.cout
        for n0, off, pc in B["proj"]:
            dense.conv(y, dataclasses.replace(pc, w=w_img[0, off:]), out=out, out_coff=n0,
                       residual=x if s.skip else None, res_coff=n0, w_img_stride=w_img.shape[1])
        self._mark("project")
        return out

    def forward_hl(self, x: torch.Tensor, r3_out: Optional[dense.HL] = None) -> Tuple[dense.HL, dense.HL]:
        """x (M, 3, H, W) fp32 images -> (reduction_3, reduction_4) as hi/lo (M, 1, h, w, .).  r3_out: optional tensor
        whose channels [0, pad_to(c3)) receive reduction_3 (e.g. the encoder heads' concat tensor)."""
        if self.training:
            raise NotImplementedError("EfficientNetTrunk runs in eval mode only")
        P = self.packed()
        M, _, H, W = x.shape
        Ho, Wo = out_size(H, 3, 2, self.stem_pad), out_size(W, 3, 2, self.stem_pad)
        self._mark("start")
        h = dense.effnet_stem(x, *P["stem"], (Ho, Wo), (self.stem_pad[0], self.stem_pad[0]))
        self._mark("stem")
        r3 = None
        for i in range(len(self._blocks)):
            h = self.forward_block(i, h, out=r3_out if i == self.endpoint else None)
            if i == self.endpoint:
                r3 = h
        return r3, h

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(M, 3, H, W) -> (reduction_3 (M, c3, H/8, W/8), reduction_4 (M, c4, H/16, W/16)) fp32 NCHW.  In train mode
        both carry a grad_fn; their memory is channels-last."""
        if self.training:
            return self.forward_train(x)
        r3, r4 = self.forward_hl(x)
        return dense.to_f32(r3).squeeze(1), dense.to_f32(r4).squeeze(1)

    def launches_per_block(self) -> List[int]:
        """Kernel launches of each block: expand chunks, depthwise + sum reduction, gate + weight scaling, projection chunks (a
        128-column chunk is one stp3_conv_fwd launch)."""
        out = []
        for blk in self._blocks:
            s = blk.spec
            out.append((len(dense.se_chunks(s.exp)) if s.exp != s.cin else 0) + 2 + 2 + len(dense.se_chunks(s.cout)))
        return out

    # ------------------------------------------------------------------------------------------------ train mode
    def forward_train(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """The train-mode forward as one autograd node: batch-statistics BatchNorm (running statistics updated with each
        module's momentum and eps; SyncBatchNorm children take the process group's statistics), drop-connect on the
        identity-skip blocks with one torch.rand of M values per block in block order.  Every trunk parameter receives
        a gradient; the images do not (a tensor that requires grad is refused)."""
        if x.requires_grad:
            raise NotImplementedError("EfficientNetTrunk (train mode): the gradient with respect to the images is not "
                                      "computed; pass images that do not require grad (e.g. x.detach())")
        if not x.is_cuda:
            raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
        for name, m in self.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                dense_train.check_bn(m, f"EfficientNetTrunk.{name}")
        params = tuple(p for p in self.parameters() if p.requires_grad)
        return _TrunkTrainFn.apply(self, x.float().contiguous(), *params)

    def _train_forward(self, x: torch.Tensor):
        """x (M, 3, H, W) -> ((reduction_3, reduction_4) channels-last fp32, tape for _train_backward).  Per block:
            _expand_conv              conv1x1_raw on the input's hi/lo planes      -> x0
            _bn0 + swish              bn_stats_module, bn_act                      -> h
            _depthwise_conv           dw_raw (the eval kernels' static pads)       -> d
            _bn1 + swish              bn_stats_module, bn_act                      -> y
            squeeze-excite            image_channel_sums, stp3_se_gate (gate only), bn_act(y * gate) -> gy (+ planes)
            _project_conv             conv_raw on gy's planes                      -> p
            _bn2 (+ drop-connect + skip)  bn_stats_module, bn_act(scale, res)      -> block output (+ planes)"""
        M, _, H, W = x.shape
        dev = x.device
        n = len(self._blocks)
        rates = drop_connect_rates(n)
        Ho, Wo = out_size(H, 3, 2, self.stem_pad), out_size(W, 3, 2, self.stem_pad)
        raw = dense_train.stem_raw(x, self._conv_stem.weight, (Ho, Wo), self.stem_pad[0])
        st = dense_train.bn_stats_module(raw, self._bn0)
        h, h_hl = dense_train.bn_act(raw, st, self._bn0, swish=True, hl=self._blocks[0].spec.exp != self._blocks[0].spec.cin)
        tape = {"x": x, "raw": raw, "st": st, "blocks": []}
        r3 = None
        for i, blk in enumerate(self._blocks):
            s: BlockSpec = blk.spec
            scale = None
            if s.skip and rates[i] > 0:
                keep = 1.0 - rates[i]
                scale = torch.floor(keep + torch.rand(M, dtype=torch.float32, device=dev)) / keep
            nxt = self._blocks[i + 1].spec if i + 1 < n else None
            h, h_hl, bt = self._train_block(blk, h, h_hl, scale, nxt is not None and nxt.exp != nxt.cin)
            tape["blocks"].append(bt)
            if i == self.endpoint:
                r3 = h
        return (r3, h), tape

    @staticmethod
    def _se_weights(blk: MBConvBlock):
        s = blk.spec
        return (blk._se_reduce.weight.detach().float().reshape(s.se, s.exp).contiguous(),
                blk._se_reduce.bias.detach().float().contiguous(),
                blk._se_expand.weight.detach().float().reshape(s.exp, s.se).contiguous(),
                blk._se_expand.bias.detach().float().contiguous())

    def _train_block(self, blk: MBConvBlock, xin: torch.Tensor, xin_hl: Optional[dense.HL], scale, out_hl: bool):
        s: BlockSpec = blk.spec
        M, H, W, _ = xin.shape
        t = {"x": xin, "scale": scale}
        h = xin
        if s.exp != s.cin:
            t["x0"] = dense_train.conv1x1_raw(xin_hl, blk._expand_conv.weight)
            t["st0"] = dense_train.bn_stats_module(t["x0"], blk._bn0)
            h, _ = dense_train.bn_act(t["x0"], t["st0"], blk._bn0, swish=True)
        Ho, Wo = out_size(H, s.k, s.stride, s.pad), out_size(W, s.k, s.stride, s.pad)
        t["h"] = h
        t["d"] = dense_train.dw_raw(h, blk._depthwise_conv.weight, s.stride, s.pad[0], (Ho, Wo))
        t["st1"] = dense_train.bn_stats_module(t["d"], blk._bn1)
        t["y"], _ = dense_train.bn_act(t["d"], t["st1"], blk._bn1, swish=True)
        t["sums"] = dense_train.image_channel_sums(t["y"])
        t["gate"] = torch.empty((M, s.exp), dtype=torch.float32, device=xin.device)
        # stp3_se_gate computes the gate; the per-image projection weights it also writes are not used here (one
        # zero row keeps them small): the projection reads the gated activation instead
        dense.se_gate(t["sums"], Ho * Wo, s.exp, *self._se_weights(blk),
                      torch.zeros((1, s.exp), dtype=torch.float32, device=xin.device), gate=t["gate"])
        t["gy"], gy_hl = dense_train.bn_act(t["y"], None, None, swish=False, mul=t["gate"], hl=True)
        t["p"] = dense_train.conv_raw(gy_hl, blk._project_conv.weight, 1)
        t["st2"] = dense_train.bn_stats_module(t["p"], blk._bn2)
        out, hl = dense_train.bn_act(t["p"], t["st2"], blk._bn2, swish=False, scale=scale,
                                     res=xin if s.skip else None, hl=out_hl)
        return out, hl, t

    def _train_backward(self, tape, g3: torch.Tensor, g4: torch.Tensor) -> dict:
        """Reverse walk of _train_forward from the endpoints' gradients (M, h, w, c) -> {parameter: gradient}."""
        grads = {}
        g = g4
        for i in reversed(range(len(self._blocks))):
            if i == self.endpoint:
                g = g + g3
            g = self._block_backward(self._blocks[i], tape["blocks"][i], g, grads)
            tape["blocks"][i] = None                # its activations are freed as the walk goes
        gz = dense_train.bn_act_grad(g, tape["raw"], tape["st"], self._bn0, swish=True)
        dz, grads[self._bn0.weight], grads[self._bn0.bias], _ = dense_train.bn_backward(gz, tape["raw"], tape["st"],
                                                                                       self._bn0.weight, None)
        grads[self._conv_stem.weight] = dense_train.stem_wgrad(tape["x"], dz, self.stem_pad[0])
        return grads

    def _block_backward(self, blk: MBConvBlock, t: dict, g: torch.Tensor, grads: dict) -> torch.Tensor:
        s: BlockSpec = blk.spec
        xin = t["x"]
        M, H, W, _ = xin.shape
        Ho, Wo = g.shape[1:3]
        gp = g if t["scale"] is None else dense_train.bn_act_grad(g, None, None, None, swish=False, scale=t["scale"])
        dp, grads[blk._bn2.weight], grads[blk._bn2.bias], _ = dense_train.bn_backward(gp, t["p"], t["st2"],
                                                                                     blk._bn2.weight, None)
        grads[blk._project_conv.weight] = dense_train.conv_wgrad(t["gy"], dp, 1, 1, 1)
        u = dense_train.conv1x1_dgrad(dp, blk._project_conv.weight)          # ungated: the gate is applied below
        # squeeze-excite: dgate = sum_p y u; the chain through sigmoid, W_e, swish and W_r; the mean's gradient and the
        # gated u enter _bn1's swish backward in the same pass
        w_r, b_r, w_e, _ = self._se_weights(blk)
        dgate = dense_train.image_channel_dot(t["y"], u)
        de, sr, dr, dmean = dense_train.se_backward(dgate, t["gate"], t["sums"], Ho * Wo, w_r, b_r, w_e)
        m = t["sums"] * (1.0 / (Ho * Wo))
        grads[blk._se_expand.weight] = dense_train.conv_wgrad(sr.view(M, 1, 1, s.se), de.view(M, 1, 1, s.exp), 1, 1, 1)
        grads[blk._se_expand.bias] = dense_train.channel_sums(de.view(M, 1, 1, s.exp))
        grads[blk._se_reduce.weight] = dense_train.conv_wgrad(m.view(M, 1, 1, s.exp), dr.view(M, 1, 1, s.se), 1, 1, 1)
        grads[blk._se_reduce.bias] = dense_train.channel_sums(dr.view(M, 1, 1, s.se))
        gd = dense_train.bn_act_grad(u, t["d"], t["st1"], blk._bn1, swish=True, mul=t["gate"], add=dmean)
        dd, grads[blk._bn1.weight], grads[blk._bn1.bias], _ = dense_train.bn_backward(gd, t["d"], t["st1"],
                                                                                     blk._bn1.weight, None)
        grads[blk._depthwise_conv.weight] = dense_train.dw_wgrad(t["h"], dd, s.k, s.stride, s.pad[0])
        dx = dense_train.dw_dgrad(dd, blk._depthwise_conv.weight, s.stride, s.pad[0], (H, W))
        if s.exp != s.cin:
            gx0 = dense_train.bn_act_grad(dx, t["x0"], t["st0"], blk._bn0, swish=True)
            dx0, grads[blk._bn0.weight], grads[blk._bn0.bias], _ = dense_train.bn_backward(gx0, t["x0"], t["st0"],
                                                                                          blk._bn0.weight, None)
            grads[blk._expand_conv.weight] = dense_train.conv_wgrad(xin, dx0, 1, 1, 1)
            dx = dense_train.conv_dgrad(dx0, blk._expand_conv.weight, 1, H, W)
        if s.skip:
            dx += g
        return dx


class _TrunkTrainFn(torch.autograd.Function):
    """The train-mode trunk as one autograd node, like the heads' (_DeepLabTrainFn): forward keeps the activations and
    statistics, backward walks the blocks in reverse on the train-mode kernels.  The backward is not itself
    differentiable, runs once per forward (retain_graph is refused), and refuses parameters modified in place between
    forward and backward.  It ignores autocast: the trunk always computes in fp32 (hi/lo operands)."""

    @staticmethod
    def forward(ctx, trunk, x, *params):
        (r3, r4), tape = trunk._train_forward(x)
        ctx.trunk, ctx.tape, ctx.params = trunk, tape, params
        ctx.versions = [p._version for p in params]
        return r3.permute(0, 3, 1, 2), r4.permute(0, 3, 1, 2)

    @staticmethod
    @once_differentiable
    def backward(ctx, g3, g4):
        if ctx.tape is None:
            raise RuntimeError("EfficientNetTrunk (train mode): backward ran a second time through the same forward; "
                               "the activations are released after the first backward (retain_graph is not "
                               "supported) -- run the forward again")
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("EfficientNetTrunk (train mode): a trunk parameter was modified in place between forward "
                               "and backward (e.g. optimizer.step() before loss.backward())")
        tape, ctx.tape = ctx.tape, None
        grads = ctx.trunk._train_backward(tape, g3.float().permute(0, 2, 3, 1).contiguous(),
                                          g4.float().permute(0, 2, 3, 1).contiguous())
        return (None, None) + tuple(grads.get(p) for p in ctx.params)
