"""TEST INFRASTRUCTURE -- a torch restatement of the efficientnet-pytorch 0.7.0 trunk (b4 / b0), usable in fp64 and fp32.

It exposes the attribute surface the reference's Encoder walks (stp3/models/encoder.py:39-86: _conv_stem, _bn0,
_swish, _blocks[i](x, drop_connect_rate=...), _global_params, and the _conv_head / _bn1 / _avg_pooling / _dropout / _fc
that delete_unused_layers removes) and efficientnet-pytorch's state-dict names.  The block table, the static "same"
padding and the block structure are restated from the package's published definition (efficientnet_params,
BlockDecoder strings, round_filters / round_repeats, Conv2dStaticSamePadding, MBConvBlock); the package itself is not
available here to compare against.  Eval mode only: drop-connect is the identity."""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

# name -> (width, depth, resolution)
GLOBAL = {'b0': (1.0, 1.0, 224), 'b4': (1.4, 1.8, 380)}
# 'r1_k3_s11_e1_i32_o16_se0.25', ... as (repeats, kernel, stride, expand, in, out)
BLOCKS_ARGS = [(1, 3, 1, 1, 32, 16), (2, 3, 2, 6, 16, 24), (2, 5, 2, 6, 24, 40), (3, 3, 2, 6, 40, 80),
               (3, 5, 1, 6, 80, 112), (4, 5, 2, 6, 112, 192), (1, 3, 1, 6, 192, 320)]
SE_RATIO, BN_EPS, BN_MOMENTUM = 0.25, 1e-3, 0.01


def _round_filters(filters, width, divisor=8):
    filters *= width
    new = max(divisor, int(filters + divisor / 2) // divisor * divisor)
    if new < 0.9 * filters:
        new += divisor
    return int(new)


def static_pad(k, s, size):
    """Conv2dStaticSamePadding: pads computed once for the nominal input size, (top/left, bottom/right)."""
    oh = math.ceil(size / s)
    p = max((oh - 1) * s + k - size, 0)
    return (p // 2, p - p // 2)


def block_table(version):
    """(stem out, stem pad, [dict(cin, exp, cout, k, s, se, pad)] for every block of the full model)."""
    width, depth, size = GLOBAL[version]
    stem_pad = static_pad(3, 2, size)
    size = math.ceil(size / 2)
    rows = []
    for r, k, s, e, i, o in BLOCKS_ARGS:
        i, o, r = _round_filters(i, width), _round_filters(o, width), int(math.ceil(depth * r))
        for j in range(r):
            cin, st = (i, s) if j == 0 else (o, 1)
            rows.append(dict(cin=cin, exp=cin * e, cout=o, k=k, s=st, se=max(1, int(cin * SE_RATIO)),
                             pad=static_pad(k, st, size)))
            if j == 0:
                size = math.ceil(size / s)
    return _round_filters(32, width), stem_pad, rows


class _SamePadConv(nn.Conv2d):
    def __init__(self, cin, cout, k, stride=1, groups=1, bias=True, pad=(0, 0)):
        super().__init__(cin, cout, k, stride=stride, groups=groups, bias=bias)
        self.pad = pad

    def forward(self, x):
        a, b = self.pad
        return super().forward(F.pad(x, (a, b, a, b)) if (a or b) else x)


def _bn(c):
    return nn.BatchNorm2d(c, momentum=BN_MOMENTUM, eps=BN_EPS)


class MBConvBlock(nn.Module):
    def __init__(self, r):
        super().__init__()
        self.r = r
        if r['exp'] != r['cin']:
            self._expand_conv = _SamePadConv(r['cin'], r['exp'], 1, bias=False)
            self._bn0 = _bn(r['exp'])
        self._depthwise_conv = _SamePadConv(r['exp'], r['exp'], r['k'], stride=r['s'], groups=r['exp'], bias=False,
                                            pad=r['pad'])
        self._bn1 = _bn(r['exp'])
        self._se_reduce = _SamePadConv(r['exp'], r['se'], 1)
        self._se_expand = _SamePadConv(r['se'], r['exp'], 1)
        self._project_conv = _SamePadConv(r['exp'], r['cout'], 1, bias=False)
        self._bn2 = _bn(r['cout'])
        self._swish = nn.SiLU()

    def forward(self, inputs, drop_connect_rate=None):
        x = inputs
        if self.r['exp'] != self.r['cin']:
            x = self._swish(self._bn0(self._expand_conv(inputs)))
        x = self._swish(self._bn1(self._depthwise_conv(x)))
        s = F.adaptive_avg_pool2d(x, 1)
        s = self._se_expand(self._swish(self._se_reduce(s)))
        x = torch.sigmoid(s) * x
        x = self._bn2(self._project_conv(x))
        if self.r['s'] == 1 and self.r['cin'] == self.r['cout']:
            x = x + inputs                 # drop_connect is the identity in eval mode
        return x


class EfficientNetOracle(nn.Module):
    """The full model's trunk (every block, plus the head layers the reference deletes)."""

    def __init__(self, version='b4'):
        super().__init__()
        stem, stem_pad, rows = block_table(version)
        self.rows = rows
        self._conv_stem = _SamePadConv(3, stem, 3, stride=2, bias=False, pad=stem_pad)
        self._bn0 = _bn(stem)
        self._blocks = nn.ModuleList(MBConvBlock(r) for r in rows)
        self._swish = nn.SiLU()
        self._global_params = SimpleNamespace(drop_connect_rate=0.2)
        head = _round_filters(1280, GLOBAL[version][0])
        self._conv_head = _SamePadConv(rows[-1]['cout'], head, 1, bias=False)
        self._bn1 = _bn(head)
        self._avg_pooling = nn.AdaptiveAvgPool2d(1)
        self._dropout = nn.Dropout(0.2)
        self._fc = nn.Linear(head, 1000)


def truncate(net, version):
    """What the reference's delete_unused_layers leaves for DOWNSAMPLE = 8."""
    last = {'b0': 10, 'b4': 21}[version]
    del net._blocks[last + 1:]
    for name in ('_conv_head', '_bn1', '_avg_pooling', '_dropout', '_fc'):
        delattr(net, name)
    return net


def endpoints(net, x):
    """reduction_3, reduction_4 exactly as the reference's get_features_depth selects them (ds = 8)."""
    x = net._swish(net._bn0(net._conv_stem(x)))
    ends, prev = [], x
    for block in net._blocks:
        x = block(x, drop_connect_rate=0.0)
        if prev.size(2) > x.size(2):
            ends.append(prev)
        prev = x
    ends.append(x)
    return ends[2], ends[3]


def init_random(net, seed=0):
    """Seeded synthetic weights with realistic scales: He-scaled convolutions, BN statistics near identity, SE biases
    that keep the gate away from saturation."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, m in net.named_modules():
            if isinstance(m, nn.Conv2d):
                fan = m.weight[0].numel()
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * math.sqrt(2.0 / fan))
                if m.bias is not None:
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
            elif isinstance(m, nn.BatchNorm2d):
                c = m.num_features
                m.weight.copy_(0.5 + 0.5 * torch.rand(c, generator=g))
                m.bias.copy_(0.1 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                m.running_var.copy_(0.5 + torch.rand(c, generator=g))
            elif isinstance(m, nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.01)
                m.bias.zero_()
    return net
