"""Native EfficientNet trunk (efficientnet-pytorch 0.7.0, b4 and b0) truncated for the ds = 8 encoder like
stp3/models/encoder.py:39-55: the stem and blocks 0..21 (b4) / 0..10 (b0), with the package's attribute names, so a
released ST-P3 checkpoint's `encoder.backbone.*` keys load with strict=True.

Eval-mode inference only.  Per MBConv block (include/stp3_b200.h):
    _expand_conv + _bn0 + swish      stp3_conv_fwd (swish), in column chunks of <= 128 output channels
    _depthwise_conv + _bn1 + swish   stp3_dw_fwd, which also emits the squeeze-excite spatial sums
    squeeze-excite                   stp3_se_gate: the gate of every image folded into per-image projection weights
    _project_conv + _bn2 (+ skip)    stp3_conv_fwd with per-image weights (and res_mode 1 for the identity skip)
BatchNorm eps is each module's own (1e-3 in the trunk).  Activations stay bf16 hi/lo planes from the stem to both
endpoints: reduction_3 (block 9 / 5 output, 1/8) and reduction_4 (block 21 / 10 output, 1/16)."""
import dataclasses
import math
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from .. import dense
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
    def __init__(self, version: str = 'b4', downsample: int = 8):
        super().__init__()
        if version not in PARAMS:
            raise NotImplementedError(f"EfficientNet-{version}: the native trunk covers b4 and b0")
        if downsample != 8:
            raise NotImplementedError("the native trunk is truncated for the ds = 8 encoder")
        self.version = version
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
        if mode:
            raise NotImplementedError("EfficientNetTrunk: the sm_90a trunk implements the eval-mode forward only "
                                      "(BatchNorm folded into the kernels); training the trunk is not supported")
        return nn.Module.train(self, False)

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
        """(M, 3, H, W) -> (reduction_3 (M, c3, H/8, W/8), reduction_4 (M, c4, H/16, W/16)) fp32 NCHW."""
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
