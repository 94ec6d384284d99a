"""Host side of the train-mode dense path (the BEV decoder, the DeepLab head and the TemporalBlocks in train(),
include/stp3_b200.h "Train mode"): convolution without folded BatchNorm (2-D, and causal 3-D on (B, T, ...) planes),
BatchNorm with batch statistics (stats / apply with dropout / backward), the input gradient of a convolution on
stp3_conv_fwd (transposed weights, mirrored taps, dilated too; stride 2 as four phase convolutions; anti-causal time
taps for the 3-D ones), the weight gradient (2-D and causal 3-D), per-image channel sums, the temporal pair mean of
the pyramid-pooling branch, and the bilinear x2 pair (dense, and on a channel window of a wider tensor).

Tensors are fp32 channels-last (N, H, W, C) contiguous; the inputs of the tensor-core convolutions are the usual
bf16 hi/lo planes (dense.HL with T = 1).  Nothing here falls back to ATen convolutions or F.batch_norm.

Autocast: a train-mode forward run under torch.autocast("cuda", dtype=torch.float16 / torch.bfloat16) takes its
precision `mode` from amp_mode() and records it; the convolutions, input gradients and weight gradients of that step
(forward and backward) then read ONE 16-bit plane per operand (dense.HL with lo None, weights rounded to the same type,
as autocast rounds the operands of F.conv2d) and issue one MMA per product, accumulating in fp32.  mode None (outside
autocast) is the fp32-equivalent hi/lo path, bit for bit.  BatchNorm statistics, running statistics and the BatchNorm
backward stay fp32 in every mode, and so do the tensors the functions return.
"""
import ctypes
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib, dense, parallel


def _p(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _f32_cl(t: torch.Tensor) -> torch.Tensor:
    assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda and t.dim() == 4, (t.dtype, t.shape)
    return t


def _row_stride(t: torch.Tensor) -> int:
    """Row stride of an fp32 (N, H, W, C) tensor whose pixel rows hold C contiguous channels at one stride: a contiguous
    tensor, or a channel slice t[..., a:b] of a wider channels-last one (the DeepLab head's concat tensor)."""
    assert t.dtype == torch.float32 and t.is_cuda and t.dim() == 4, (t.dtype, t.shape)
    N, H, W, C = t.shape
    cs = t.stride(2)
    assert t.stride(3) == 1 and t.stride(1) == W * cs and t.stride(0) == H * W * cs and C <= cs, t.stride()
    return cs


def amp_mode() -> Optional[torch.dtype]:
    """The precision mode of a train-mode forward: torch.float16 / torch.bfloat16 inside a CUDA autocast region of that
    type, None (fp32-equivalent hi/lo operands) outside one."""
    if not torch.is_autocast_enabled("cuda"):
        return None
    dt = torch.get_autocast_dtype("cuda")
    return dt if dt in dense.PLANE_OPERAND else None


def amp_kw(mode: Optional[torch.dtype]) -> dict:
    """The keyword arguments that select `mode` in to_hl, bn_apply, conv_dgrad and conv_wgrad: none outside autocast,
    so the fp32 path makes exactly the calls it always made, and a function that has no `mode` parameter is never
    handed one.  The launch-by-launch contract suites replace to_hl, bn_apply and conv_wgrad with recorders that take
    `mode` as a keyword and record fp32 and autocast steps alike."""
    return {} if mode is None else {"mode": mode}


def operand(t: torch.Tensor, mode: Optional[torch.dtype]):
    """What conv_dgrad / conv_wgrad read: t itself outside autocast; under a mode, ONE plane of t (to_hl), so a
    gradient that feeds both the input and the weight gradient is converted once.  A one-plane HL passes through."""
    if mode is None or isinstance(t, dense.HL):
        return t
    return to_hl(t.reshape(-1, *t.shape[-3:]).contiguous(), mode=mode)


def _dims(t) -> Tuple[int, int, int, int, int]:
    """(images, H, W, channels, row stride) of an fp32 (N, H, W, C) / (B, T, H, W, C) tensor or a one-plane HL"""
    if isinstance(t, dense.HL):
        return t.hi.shape[0] * t.hi.shape[1], t.hi.shape[2], t.hi.shape[3], t.c, t.hi.shape[-1]
    return t.numel() // (t.shape[-3] * t.shape[-2] * t.shape[-1]), t.shape[-3], t.shape[-2], t.shape[-1], t.shape[-1]


def _plane_empty(N: int, H: int, W: int, cp: int, mode: torch.dtype, dev) -> dense.HL:
    return dense.HL(torch.empty((N, 1, H, W, cp), dtype=mode, device=dev), None, 0)


def to_hl(x: torch.Tensor, cp: Optional[int] = None, mode: Optional[torch.dtype] = None) -> dense.HL:
    """(N, H, W, C) fp32 -> HL (N, 1, H, W, cp) bf16 hi/lo planes, padding channels zero.  mode (torch.float16 /
    torch.bfloat16): ONE plane of that type instead (lo None), x rounded to nearest even, overflow to +-inf
    (stp3_f32_to_plane)."""
    _f32_cl(x)
    N, H, W, C = x.shape
    if mode is not None:
        out = _plane_empty(N, H, W, cp or dense.pad_to(C), mode, x.device)
        out.c = C
        with torch.cuda.device(x.device):
            code = _lib.lib().stp3_f32_to_plane(x.data_ptr(), 1, N, C, H, W, out.hi.shape[-1], dense.PLANE_OPERAND[mode],
                                                out.hi.data_ptr(), _stream(x.device))
        _lib.check(code, "stp3_f32_to_plane")
        return out
    out = dense.HL.empty(N, 1, H, W, C, x.device, cp=cp)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_f32_to_hilo(x.data_ptr(), 1, N, C, H, W, out.hi.shape[-1], out.hi.data_ptr(),
                                           out.lo.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_f32_to_hilo")
    return out


# ------------------------------------------------------------------------------------------------ convolutions
def _pack_taps(mats: List[torch.Tensor], taps: List[Tuple[int, ...]], cin: int, cout: int,
               plane: Optional[torch.dtype] = None) -> dense.PackedConv:
    """Weight matrices (cout, cin) of arbitrary (dy, dx) or (dt, dy, dx) taps -> the tap-major / K-major layout of
    stp3_conv_fwd (plane: one plane of that 16-bit type, stp3_conv_fwd_plane)."""
    cin_p, bn = dense.pad_to(cin), dense.out_tile(cout)
    dev = mats[0].device
    m = torch.zeros((len(mats), bn, cin_p), dtype=torch.float32, device=dev)
    for i, w in enumerate(mats):
        m[i, :cout, :cin] = w
    packed = dense.pack_planes(m, plane)
    bias = torch.zeros(bn, dtype=torch.float32, device=dev)
    dense._PACK_COUNTER += 1
    return dense.PackedConv(packed, bias, [tuple(t) if len(t) == 3 else (0, *t) for t in taps], cin_p, bn, cout, 1, 0,
                            cin_p, dense._PACK_COUNTER, plane)


def dgrad_taps(kh: int, kw: int, stride: int, pad: int, dilation: int = 1):
    """Input gradient of y[o] = sum_t W_t x[o*stride + d_t] as stride-1 convolutions of the output gradient G:
    a list of ((py, px), [(ky, kx, ey, ex)]) -- phase (py, px) of the input (every pixel for stride 1) receives
    sum over the listed taps of W[:, :, ky, kx]^T G[i + ey, j + ex].  Stride 1: e = -d (d = k * dilation - pad).
    Stride 2 (undilated): input pixel 2i + py is read by tap d when py - d is even, from output i + (py - d) / 2."""
    if dilation < 1:
        raise ValueError(f"dilation must be >= 1, got {dilation}")
    if stride == 1:
        return [((0, 0), [(ky, kx, pad - ky * dilation, pad - kx * dilation) for ky in range(kh) for kx in range(kw)])]
    if dilation != 1:
        raise NotImplementedError("input gradient of a dilated stride-2 convolution")
    phases = []
    for py in range(2):
        for px in range(2):
            taps = [(ky, kx, (py - (ky - pad)) // 2, (px - (kx - pad)) // 2) for ky in range(kh) for kx in range(kw)
                    if (py - (ky - pad)) % 2 == 0 and (px - (kx - pad)) % 2 == 0]
            phases.append(((py, px), taps))
    return phases


def dgrad_taps_3d(kt: int, kh: int, kw: int):
    """Input gradient of the causal y[t, p] = sum W_k x[t + it - (kt-1), p + (ky, kx) - pad] (stride 1, 'same' spatial
    padding, pad = (kh-1)//2 = (kw-1)//2) as one convolution of the output gradient G: [(it, ky, kx, et, ey, ex)], x
    receives sum over the list of W[:, :, it, ky, kx]^T G[t + et, p + (ey, ex)].  et = (kt-1) - it >= 0 (anti-causal:
    frames at or past T are zero padding), ey = pad - ky, ex = pad - kx."""
    if kh != kw or kh % 2 != 1:
        raise ValueError(f"the spatial kernel must be square and odd, got {kh}x{kw}")
    pad = (kh - 1) // 2
    return [(it, ky, kx, kt - 1 - it, pad - ky, pad - kx) for it in range(kt) for ky in range(kh) for kx in range(kw)]


def pack_dgrad3d(weight: torch.Tensor, plane: Optional[torch.dtype] = None) -> dense.PackedConv:
    """weight (cout, cin, kt, kh, kw) of a causal 3-D convolution -> the transposed (cin x cout) tap matrices with the
    anti-causal taps of dgrad_taps_3d, for stp3_conv_fwd on the output gradient."""
    w = weight.detach().float()
    cout, cin, kt, kh, kw = w.shape
    taps = dgrad_taps_3d(kt, kh, kw)
    return _pack_taps([w[:, :, it, ky, kx].t() for it, ky, kx, _, _, _ in taps], [t[3:] for t in taps], cout, cin, plane)


def pack_dgrad(weight: torch.Tensor, stride: int, pad: int, dilation: int = 1, plane: Optional[torch.dtype] = None):
    """weight (cout, cin, kh, kw) -> [((py, px), PackedConv or None)]: the transposed (cin x cout) tap matrices of every
    phase, for stp3_conv_fwd on the output gradient."""
    w = weight.detach().float()
    cout, cin, kh, kw = w.shape
    out = []
    for ph, taps in dgrad_taps(kh, kw, stride, pad, dilation):
        if not taps:
            out.append((ph, None))
            continue
        mats = [w[:, :, ky, kx].t() for ky, kx, _, _ in taps]
        out.append((ph, _pack_taps(mats, [(ey, ex) for _, _, ey, ex in taps], cout, cin, plane)))
    return out


def conv_raw(x: dense.HL, weight: torch.Tensor, stride: int, bias: Optional[torch.Tensor] = None,
             sigmoid: bool = False, nchw: bool = False, dilation: int = 1,
             img_bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Convolution without folded BatchNorm ('same' zero padding, like every decoder and DeepLab convolution) on
    stp3_conv_fwd: (N, Ho, Wo, cout) fp32 channels-last, or (N, cout, Ho, Wo) with nchw (the reference's logits layout,
    optional sigmoid), N = B*T images of x (B, T, H, W, .).  A 5-D weight (cout, cin, kt, kh, kw) is the causal 3-D
    convolution of the TemporalBlocks (time padded on the left, stride 1).  img_bias (N, out_tile(cout)) replaces the
    bias per image.  A one-plane x (to_hl / bn_apply with a mode) runs the one-product convolution on the weights
    rounded to x's type."""
    cout = weight.shape[0]
    b = bias.detach().float() if bias is not None else torch.zeros(cout, device=weight.device)
    plane = x.hi.dtype if x.lo is None else None
    pc = dense.pack_conv(weight.detach().float(), b, stride=stride, dilation=dilation, plane=plane)
    B, T, H, W, _ = x.hi.shape
    N = B * T
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    if nchw:
        out = torch.empty((N, cout, Ho, Wo), dtype=torch.float32, device=x.hi.device)
    else:
        out = torch.empty((N, Ho, Wo, cout), dtype=torch.float32, device=x.hi.device)
    dense.conv(x, pc, out_f32=out, n_valid=cout, out_f32_nhwc=not nchw, sigmoid=sigmoid, store=False, tune=(0, 0),
               img_bias=img_bias)
    return out


def conv_dgrad(g: torch.Tensor, weight: torch.Tensor, stride: int, H: int, W: int,
               packed=None, dilation: int = 1, img_bias: Optional[torch.Tensor] = None, T: int = 1,
               mode: Optional[torch.dtype] = None) -> torch.Tensor:
    """dL/dx (N, H, W, cin) of a 'same'-padded convolution from g = dL/dy (N, Ho, Wo, cout).  Stride 1 only: img_bias
    (N, out_tile(cin)) is added to every pixel of image n (a spatially constant gradient term, for free).  A 5-D weight
    (cout, cin, kt, kh, kw) is the causal 3-D convolution of conv_raw on N = B*T frames (T given): its input gradient is
    one stp3_conv_fwd with the anti-causal taps of dgrad_taps_3d.  mode (the forward's amp_mode()): g and the weights
    as one plane of that type, one product each; g may then be its plane already (operand())."""
    if isinstance(g, dense.HL):
        assert mode is not None and g.lo is None and g.hi.dtype == mode
    else:
        _f32_cl(g)
    N, cout, dev = _dims(g)[0], _dims(g)[3], (g.hi if isinstance(g, dense.HL) else g).device
    if weight.dim() == 5:
        cin = weight.shape[1]
        assert N % T == 0 and stride == 1 and dilation == 1
        pc = packed if packed is not None else pack_dgrad3d(weight, mode)
        g_hl = operand(g, mode) if mode is not None else to_hl(g)
        g_hl = dense.HL(g_hl.hi.view(N // T, T, *g_hl.hi.shape[2:]),
                        g_hl.lo.view(N // T, T, *g_hl.lo.shape[2:]) if g_hl.lo is not None else None, cout)
        out = torch.empty((N, H, W, cin), dtype=torch.float32, device=dev)
        dense.conv(g_hl, pc, out_f32=out, n_valid=cin, out_f32_nhwc=True, out_hw=(H, W), store=False, tune=(0, 0),
                   img_bias=img_bias)
        return out
    cout, cin, kh, kw = weight.shape
    pad = (kh - 1) * dilation // 2
    packed = packed if packed is not None else pack_dgrad(weight, stride, pad, dilation, mode)
    g_hl = operand(g, mode) if mode is not None else to_hl(g)
    if stride == 1:
        out = torch.empty((N, H, W, cin), dtype=torch.float32, device=dev)
        dense.conv(g_hl, packed[0][1], out_f32=out, n_valid=cin, out_f32_nhwc=True, out_hw=(H, W), store=False,
                   tune=(0, 0), img_bias=img_bias)
        return out
    assert img_bias is None
    phases = []
    for (py, px), pc in packed:
        if pc is None:
            phases.append(None)
            continue
        Hp, Wp = (H - py + 1) // 2, (W - px + 1) // 2
        t = torch.empty((N, Hp, Wp, cin), dtype=torch.float32, device=dev)
        dense.conv(g_hl, pc, out_f32=t, n_valid=cin, out_f32_nhwc=True, out_hw=(Hp, Wp), store=False, tune=(0, 0))
        phases.append(t)
    return phase_interleave(phases, H, W)


def phase_interleave(phases: List[Optional[torch.Tensor]], H: int, W: int) -> torch.Tensor:
    """The four phases (py, px) = (0,0), (0,1), (1,0), (1,1) of a stride-2 input gradient, phase (py, px) of size
    (N, (H - py + 1) // 2, (W - px + 1) // 2, C) or None (zeros) -> (N, H, W, C) (stp3_phase_interleave)."""
    ref = next(t for t in phases if t is not None)
    N, C, dev = ref.shape[0], ref.shape[-1], ref.device
    out = torch.empty((N, H, W, C), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_phase_interleave(*[_p(t) for t in phases], N, H, W, C, out.data_ptr(), _stream(dev))
    _lib.check(code, "stp3_phase_interleave")
    return out


def conv_wgrad(x: torch.Tensor, g: torch.Tensor, kh: int, kw: int, stride: int, dilation: int = 1,
               kt: Optional[int] = None, mode: Optional[torch.dtype] = None) -> torch.Tensor:
    """dL/dW (cout, cin, kh, kw) of a 'same'-padded convolution: x (N, H, W, cin) its input, g (N, Ho, Wo, cout).
    x and g 5-D (B, T, H, W, .) with kt: the causal 3-D convolution of conv_raw, dL/dW (cout, cin, kt, kh, kw)
    (stp3_conv3d_wgrad).  mode (the forward's amp_mode()): the one-product weight gradient on x and g rounded to one
    plane of that type (stp3_conv_wgrad_plane / stp3_conv3d_wgrad_plane); either may then be its plane already
    (operand(), or the plane the forward convolution read), of N = B*T images for the 3-D one."""
    if mode is not None:
        return _conv_wgrad_plane(x, g, kh, kw, stride, dilation, kt, mode)
    L = _lib.lib()
    if x.dim() == 5:
        assert kt is not None and stride == 1 and dilation == 1 and x.shape[:4] == g.shape[:4]
        assert x.is_contiguous() and g.is_contiguous() and x.dtype == g.dtype == torch.float32
        B, T, H, W, cin = x.shape
        cout = g.shape[-1]
        nbytes = L.stp3_conv3d_wgrad_scratch_bytes(B, T, H, W, cout, cin, kt, kh, kw)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        dw = torch.empty((cout, cin, kt, kh, kw), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            code = L.stp3_conv3d_wgrad(x.data_ptr(), B, T, H, W, cin, cin, g.data_ptr(), cout, cout, kt, kh, kw,
                                       scratch.data_ptr(), nbytes, dw.data_ptr(), _stream(x.device))
        _lib.check(code, "stp3_conv3d_wgrad")
        return dw
    _f32_cl(x), _f32_cl(g)
    N, H, W, cin = x.shape
    _, Ho, Wo, cout = g.shape
    nbytes = L.stp3_conv_wgrad_scratch_bytes(N, Ho, Wo, cout, cin, kh, kw, dilation)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    dw = torch.empty((cout, cin, kh, kw), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = L.stp3_conv_wgrad(x.data_ptr(), N, H, W, cin, cin, g.data_ptr(), Ho, Wo, cout, cout, kh, kw, stride,
                                 (kh - 1) * dilation // 2, dilation, scratch.data_ptr(), nbytes, dw.data_ptr(),
                                 _stream(x.device))
    _lib.check(code, "stp3_conv_wgrad")
    return dw


def _conv_wgrad_plane(x, g, kh: int, kw: int, stride: int, dilation: int, kt: Optional[int],
                      mode: torch.dtype) -> torch.Tensor:
    L = _lib.lib()
    op = dense.PLANE_OPERAND[mode]
    fp32 = [t for t in (x, g) if not isinstance(t, dense.HL)]
    B_T = fp32[0].shape[:2] if fp32 and fp32[0].dim() == 5 else None
    xp, gp = operand(x, mode), operand(g, mode)
    for t in (xp, gp):
        assert t.lo is None and t.hi.dtype == mode, "one-plane operands of the autocast type"
    N, H, W, cin, xcs = _dims(xp)
    Ng, Ho, Wo, cout, gcs = _dims(gp)
    assert N == Ng
    dev = xp.hi.device
    if kt is not None:
        assert B_T is not None and stride == 1 and dilation == 1 and (Ho, Wo) == (H, W), "3-D: x or g (B, T, H, W, C)"
        B, T = B_T
        nbytes = L.stp3_conv3d_wgrad_scratch_bytes(B, T, H, W, cout, cin, kt, kh, kw)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        dw = torch.empty((cout, cin, kt, kh, kw), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            code = L.stp3_conv3d_wgrad_plane(op, xp.hi.data_ptr(), B, T, H, W, xcs, cin, gp.hi.data_ptr(), gcs, cout,
                                             kt, kh, kw, scratch.data_ptr(), nbytes, dw.data_ptr(), _stream(dev))
        _lib.check(code, "stp3_conv3d_wgrad_plane")
        return dw
    nbytes = L.stp3_conv_wgrad_scratch_bytes(N, Ho, Wo, cout, cin, kh, kw, dilation)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dw = torch.empty((cout, cin, kh, kw), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        code = L.stp3_conv_wgrad_plane(op, xp.hi.data_ptr(), N, H, W, xcs, cin, gp.hi.data_ptr(), Ho, Wo, gcs, cout,
                                       kh, kw, stride, (kh - 1) * dilation // 2, dilation, scratch.data_ptr(), nbytes,
                                       dw.data_ptr(), _stream(dev))
    _lib.check(code, "stp3_conv_wgrad_plane")
    return dw


# ------------------------------------------------------------------------------------------------ BatchNorm
def check_bn(bn: nn.Module, owner: str):
    """The train-mode kernels implement nn.BatchNorm2d / nn.BatchNorm3d (the TemporalBlocks') with running statistics
    and a fixed momentum, and nn.SyncBatchNorm (statistics over its process group) once torch.distributed is up."""
    if isinstance(bn, nn.SyncBatchNorm):
        if not (dist.is_available() and dist.is_initialized()):
            raise NotImplementedError(f"{owner}: SyncBatchNorm (sync_batchnorm=True / DDP) needs torch.distributed: "
                                      "init the process group before training, or use plain BatchNorm2d / BatchNorm3d")
    elif not isinstance(bn, (nn.BatchNorm2d, nn.BatchNorm3d)):
        raise NotImplementedError(f"{owner}: expected nn.BatchNorm2d or nn.BatchNorm3d, got {type(bn).__name__}")
    if not bn.track_running_stats or bn.running_mean is None:
        raise NotImplementedError(f"{owner}: BatchNorm2d(track_running_stats=False) is not supported in train mode")
    if bn.momentum is None:
        raise NotImplementedError(f"{owner}: BatchNorm2d(momentum=None) (cumulative average) is not supported in "
                                  "train mode")
    if not bn.affine:
        raise NotImplementedError(f"{owner}: BatchNorm2d(affine=False) is not supported in train mode")


def bn_group(bn: nn.Module):
    """The process group whose batch a SyncBatchNorm's statistics span (its process_group, None meaning WORLD), or
    None: plain BatchNorm, or a group of one rank, whose statistics are the local ones bit for bit."""
    if not isinstance(bn, nn.SyncBatchNorm) or not dist.is_initialized():
        return None
    group = bn.process_group if bn.process_group is not None else dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


def sync_world(bn: nn.Module, n_local: int, owner: str) -> int:
    """Ranks over which bn's batch statistics are taken (1: local statistics).  Under SyncBatchNorm every rank must hold
    at least one image, so the group's batch is at least n_local * world when n_local >= 1: the batch-of-one checks
    use that count, like torch's SyncBatchNorm."""
    group = bn_group(bn)
    if group is None:
        return 1
    if n_local < 1:
        raise ValueError(f"{owner} (train mode, SyncBatchNorm): this rank holds no images; every rank of the process "
                         "group must train on at least one")
    return dist.get_world_size(group)


@dataclass
class BNStats:
    mean: torch.Tensor
    var: torch.Tensor          # biased
    invstd: torch.Tensor
    n: int                     # rows of this rank
    group: object = None       # SyncBatchNorm: the process group the statistics span
    counts: Optional[torch.Tensor] = None      # its ranks' row counts, a pinned host copy made after the exchange ...
    counts_ready: Optional[torch.cuda.Event] = None    # ... and the event that completes it

    @property
    def n_total(self) -> int:
        """Rows over the process group: what the backward normalises its merged sums by."""
        if self.group is None:
            return self.n
        self.counts_ready.synchronize()        # recorded in the forward: long done by the backward
        return int(self.counts.sum().item())


def _bn_scratch(n_pix: int, C: int, dev) -> Tuple[torch.Tensor, int]:
    nbytes = _lib.lib().stp3_bn_scratch_bytes(n_pix, C)
    return torch.empty(nbytes, dtype=torch.uint8, device=dev), nbytes


def bn_stats(x: torch.Tensor, eps: float, momentum: float, running_mean: Optional[torch.Tensor] = None,
             running_var: Optional[torch.Tensor] = None) -> BNStats:
    """Batch mean / biased variance per channel of x (N, H, W, C); updates the running statistics when given."""
    _f32_cl(x)
    C = x.shape[-1]
    n = x.numel() // C
    dev = x.device
    mean, var, invstd = (torch.empty(C, dtype=torch.float32, device=dev) for _ in range(3))
    for t in (running_mean, running_var):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == C)
    scratch, nbytes = _bn_scratch(n, C, dev)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_bn_stats(x.data_ptr(), n, C, C, float(eps), float(momentum), _p(running_mean),
                                        _p(running_var), mean.data_ptr(), var.data_ptr(), invstd.data_ptr(),
                                        scratch.data_ptr(), nbytes, _stream(dev))
    _lib.check(code, "stp3_bn_stats")
    return BNStats(mean, var, invstd, n)


def bn_stats_module(x: torch.Tensor, bn: nn.BatchNorm2d) -> BNStats:
    """bn_stats with the module's own eps / momentum; updates its running_mean / running_var / num_batches_tracked.
    A SyncBatchNorm over more than one rank takes the statistics of the group's batch: each rank's fp64 moments record
    (stp3_bn_local_moments, into its row of the gather buffer), one all-gather, and the same merge on every rank
    (stp3_bn_merge_finalize), so every rank gets the same statistics and running-statistic bits."""
    group = bn_group(bn)
    st = bn_stats(x, bn.eps, bn.momentum, bn.running_mean, bn.running_var) if group is None else \
        _bn_stats_sync(x, bn, group)
    bn.num_batches_tracked.add_(1)
    return st


def _bn_stats_sync(x: torch.Tensor, bn: nn.SyncBatchNorm, group) -> BNStats:
    _f32_cl(x)
    C = x.shape[-1]
    n = x.numel() // C
    dev = x.device
    ws, rank = dist.get_world_size(group), dist.get_rank(group)
    rec = torch.empty((ws, 4, C), dtype=torch.float64, device=dev)
    mean, var, invstd = (torch.empty(C, dtype=torch.float32, device=dev) for _ in range(3))
    scratch, nbytes = _bn_scratch(n, C, dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        code = L.stp3_bn_local_moments(x.data_ptr(), n, C, C, rec[rank].data_ptr(), scratch.data_ptr(), nbytes,
                                       _stream(dev))
        _lib.check(code, "stp3_bn_local_moments")
        parallel.all_gather_rows(rec, group)
        code = L.stp3_bn_merge_finalize(rec.data_ptr(), ws, C, float(bn.eps), float(bn.momentum),
                                        bn.running_mean.data_ptr(), bn.running_var.data_ptr(), mean.data_ptr(),
                                        var.data_ptr(), invstd.data_ptr(), _stream(dev))
        _lib.check(code, "stp3_bn_merge_finalize")
        counts = torch.empty(ws, dtype=torch.float64, pin_memory=True)
        counts.copy_(rec[:, 0, 0], non_blocking=True)
        ready = torch.cuda.Event()
        ready.record()
    return BNStats(mean, var, invstd, n, group, counts, ready)


def bn_apply(x: torch.Tensor, st: BNStats, gamma: torch.Tensor, beta: torch.Tensor, relu: bool,
             res: Optional[torch.Tensor] = None, hl: bool = True, dropout: Tuple[float, int, int] = (0.0, 0, 0),
             y_out: Optional[torch.Tensor] = None,
             mode: Optional[torch.dtype] = None) -> Tuple[torch.Tensor, Optional[dense.HL]]:
    """y = relu?(xhat * gamma + beta (+ res)) [* keep / (1 - p)] -> (fp32 (N, H, W, C), HL planes for the next
    convolution or None).  dropout = (p, seed, offset): the keep bits of stp3_bn_apply.  y_out: where y goes (default a
    new tensor; a channel slice of a wider channels-last tensor is fine).  mode (torch.float16 / torch.bfloat16): the
    planes are ONE plane of that type (stp3_bn_apply_plane), y and the dropout bits unchanged."""
    _f32_cl(x)
    N, H, W, C = x.shape
    dev = x.device
    y = torch.empty_like(x) if y_out is None else y_out
    assert y.shape == x.shape
    y_cs = _row_stride(y)
    p, seed, offset = dropout
    if hl and mode is not None:
        out = _plane_empty(N, H, W, dense.pad_to(C), mode, dev)
        out.c = C
    else:
        out = dense.HL.empty(N, 1, H, W, C, dev) if hl else None
    g, b = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
    if res is not None:
        _f32_cl(res)
        assert res.shape == x.shape
    with torch.cuda.device(dev):
        if out is not None and out.lo is None:
            code = _lib.lib().stp3_bn_apply_plane(x.data_ptr(), N * H * W, C, C, st.mean.data_ptr(), st.invstd.data_ptr(),
                                                  g.data_ptr(), b.data_ptr(), _p(res), C, int(relu), float(p), int(seed),
                                                  int(offset), y.data_ptr(), y_cs, out.hi.data_ptr(), out.hi.shape[-1],
                                                  dense.PLANE_OPERAND[mode], _stream(dev))
            _lib.check(code, "stp3_bn_apply_plane")
            return y, out
        code = _lib.lib().stp3_bn_apply(x.data_ptr(), N * H * W, C, C, st.mean.data_ptr(), st.invstd.data_ptr(),
                                        g.data_ptr(), b.data_ptr(), _p(res), C, int(relu), float(p), int(seed),
                                        int(offset), y.data_ptr(), y_cs,
                                        _p(out.hi if out else None), _p(out.lo if out else None),
                                        out.hi.shape[-1] if out else 0, _stream(dev))
    _lib.check(code, "stp3_bn_apply")
    return y, out


def channel_sums(g: torch.Tensor) -> torch.Tensor:
    """sum over pixels per channel of g (N, H, W, C): the gradient of a convolution bias."""
    _f32_cl(g)
    C = g.shape[-1]
    n = g.numel() // C
    out = torch.empty(C, dtype=torch.float32, device=g.device)
    scratch, nbytes = _bn_scratch(n, C, g.device)
    with torch.cuda.device(g.device):
        code = _lib.lib().stp3_bn_bwd_reduce(g.data_ptr(), C, None, 0, None, 0, None, None, n, C, out.data_ptr(), None,
                                             scratch.data_ptr(), nbytes, _stream(g.device))
    _lib.check(code, "stp3_bn_bwd_reduce")
    return out


def bn_backward(g: torch.Tensor, x: torch.Tensor, st: BNStats, gamma: torch.Tensor, y_mask: Optional[torch.Tensor],
                want_masked: bool = False, dx_out: Optional[torch.Tensor] = None):
    """Backward of y = relu?(BN_batch(x) (+ res)): g = dL/dy, y_mask = the forward output y when a ReLU follows (after
    dropout, y > 0 marks the kept positive elements; the 1 / (1 - p) factor is the caller's).  g, x and y_mask may be
    channel slices of wider channels-last tensors; so may dx_out, where dL/dx goes (default a new tensor).
    -> (dL/dx, dgamma, dbeta, g masked by the ReLU (the gradient of the residual) or None)."""
    g_cs, x_cs = _row_stride(g), _row_stride(x)
    y_cs = _row_stride(y_mask) if y_mask is not None else 0
    N, H, W, C = x.shape
    n = N * H * W
    dev = x.device
    sum_g = torch.empty(C, dtype=torch.float32, device=dev)
    sum_gx = torch.empty(C, dtype=torch.float32, device=dev)
    scratch, nbytes = _bn_scratch(n, C, dev)
    gm = torch.empty((N, H, W, C), dtype=torch.float32, device=dev) if want_masked else None
    dx = torch.empty((N, H, W, C), dtype=torch.float32, device=dev) if dx_out is None else dx_out
    assert dx.shape == x.shape
    dx_cs = _row_stride(dx)
    gam = gamma.detach().float().contiguous()
    L = _lib.lib()
    if st.group is not None:
        _bn_backward_sync(g, g_cs, y_mask, y_cs, x, x_cs, st, gam, sum_g, sum_gx, scratch, nbytes, dx, dx_cs, gm)
        return dx, sum_gx, sum_g, gm
    with torch.cuda.device(dev):
        code = L.stp3_bn_bwd_reduce(g.data_ptr(), g_cs, _p(y_mask), y_cs, x.data_ptr(), x_cs, st.mean.data_ptr(),
                                    st.invstd.data_ptr(), n, C, sum_g.data_ptr(), sum_gx.data_ptr(), scratch.data_ptr(),
                                    nbytes, _stream(dev))
        _lib.check(code, "stp3_bn_bwd_reduce")
        code = L.stp3_bn_bwd_apply(g.data_ptr(), g_cs, _p(y_mask), y_cs, x.data_ptr(), x_cs, st.mean.data_ptr(),
                                   st.invstd.data_ptr(), gam.data_ptr(), sum_g.data_ptr(), sum_gx.data_ptr(), n, C,
                                   dx.data_ptr(), dx_cs, _p(gm), C, _stream(dev))
    _lib.check(code, "stp3_bn_bwd_apply")
    return dx, sum_gx, sum_g, gm


def _bn_backward_sync(g, g_cs, y_mask, y_cs, x, x_cs, st: BNStats, gam, sum_g, sum_gx, scratch, nbytes, dx, dx_cs, gm):
    """bn_backward of a SyncBatchNorm: sum_g / sum_gx (dbeta / dgamma) stay this rank's own sums, as torch's
    SyncBatchNorm returns them (DDP averages them with every other gradient); dx uses the group's sums and row count."""
    C, n, dev = x.shape[-1], st.n, x.device
    ws, rank = dist.get_world_size(st.group), dist.get_rank(st.group)
    rec = torch.empty((ws, 2, C), dtype=torch.float64, device=dev)
    tot_g, tot_gx = (torch.empty(C, dtype=torch.float32, device=dev) for _ in range(2))
    L = _lib.lib()
    with torch.cuda.device(dev):
        code = L.stp3_bn_bwd_local_sums(g.data_ptr(), g_cs, _p(y_mask), y_cs, x.data_ptr(), x_cs, st.mean.data_ptr(),
                                        st.invstd.data_ptr(), n, C, rec[rank].data_ptr(), scratch.data_ptr(), nbytes,
                                        _stream(dev))
        _lib.check(code, "stp3_bn_bwd_local_sums")
        code = L.stp3_bn_bwd_merge_sums(rec[rank].data_ptr(), 1, C, sum_g.data_ptr(), sum_gx.data_ptr(), _stream(dev))
        _lib.check(code, "stp3_bn_bwd_merge_sums")
        parallel.all_gather_rows(rec, st.group)
        code = L.stp3_bn_bwd_merge_sums(rec.data_ptr(), ws, C, tot_g.data_ptr(), tot_gx.data_ptr(), _stream(dev))
        _lib.check(code, "stp3_bn_bwd_merge_sums")
        code = L.stp3_bn_bwd_apply_global(g.data_ptr(), g_cs, _p(y_mask), y_cs, x.data_ptr(), x_cs, st.mean.data_ptr(),
                                          st.invstd.data_ptr(), gam.data_ptr(), tot_g.data_ptr(), tot_gx.data_ptr(), n,
                                          st.n_total, C, dx.data_ptr(), dx_cs, _p(gm), C, _stream(dev))
    _lib.check(code, "stp3_bn_bwd_apply_global")


def image_channel_sums(x: torch.Tensor) -> torch.Tensor:
    """(N, C) fp32 sums over the H*W pixels of every image of x (N, H, W, C), in a fixed order (stp3_image_channel_sums)."""
    _f32_cl(x)
    N, H, W, C = x.shape
    L = _lib.lib()
    nbytes = L.stp3_image_channel_sums_scratch_bytes(N, H * W, C)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.empty((N, C), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = L.stp3_image_channel_sums(x.data_ptr(), N, H * W, C, C, out.data_ptr(), scratch.data_ptr(), nbytes,
                                         _stream(x.device))
    _lib.check(code, "stp3_image_channel_sums")
    return out


def temporal_pair_mean(m: torch.Tensor, T: int, adjoint: bool = False) -> torch.Tensor:
    """The time part of a TemporalBlock's pyramid pooling (stp3_temporal_pair_mean): per-frame means m (B*T, C) -> the
    B*(T+1) pooled frames (frame t: m[0] at t = 0, (m[t-1] + m[t]) / 2 for t < T, m[T-1] at t = T); adjoint: a gradient
    (B*(T+1), C) -> (B*T, C)."""
    assert m.dtype == torch.float32 and m.is_contiguous() and m.is_cuda and m.dim() == 2
    B = m.shape[0] // (T + 1 if adjoint else T)
    assert m.shape[0] == B * (T + 1 if adjoint else T)
    out = torch.empty((B * (T if adjoint else T + 1), m.shape[1]), dtype=torch.float32, device=m.device)
    with torch.cuda.device(m.device):
        code = _lib.lib().stp3_temporal_pair_mean(m.data_ptr(), B, T, m.shape[1], int(adjoint), out.data_ptr(),
                                                  _stream(m.device))
    _lib.check(code, "stp3_temporal_pair_mean")
    return out


# ------------------------------------------------------------------------------------------------ elementwise
def upsample2x(x: torch.Tensor) -> torch.Tensor:
    """bilinear x2, align_corners=False: (N, h, w, C) -> (N, 2h, 2w, C)."""
    _f32_cl(x)
    N, h, w, C = x.shape
    y = torch.empty((N, 2 * h, 2 * w, C), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_upsample2x_f32(x.data_ptr(), N, h, w, C, y.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_upsample2x_f32")
    return y


def upsample2x_backward(gy: torch.Tensor) -> torch.Tensor:
    """Adjoint of upsample2x: (N, 2h, 2w, C) -> (N, h, w, C)."""
    _f32_cl(gy)
    N, H2, W2, C = gy.shape
    assert H2 % 2 == 0 and W2 % 2 == 0
    gx = torch.empty((N, H2 // 2, W2 // 2, C), dtype=torch.float32, device=gy.device)
    with torch.cuda.device(gy.device):
        code = _lib.lib().stp3_upsample2x_bwd(gy.data_ptr(), N, H2 // 2, W2 // 2, C, gx.data_ptr(), _stream(gy.device))
    _lib.check(code, "stp3_upsample2x_bwd")
    return gx


def upsample2x_into(x: torch.Tensor, y: torch.Tensor, coff: int) -> torch.Tensor:
    """upsample2x of x (N, h, w, C) written into channels [coff, coff + C) of the wider channels-last y (N, 2h, 2w, Cy)
    (UpsamplingConcat's concat tensor: no torch.cat); the other channels of y are not touched."""
    _f32_cl(x), _f32_cl(y)
    N, h, w, C = x.shape
    assert tuple(y.shape[:3]) == (N, 2 * h, 2 * w) and 0 <= coff and coff + C <= y.shape[3], (x.shape, y.shape, coff)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_upsample2x_window_f32(x.data_ptr(), N, h, w, C, y.data_ptr(), y.shape[3], coff,
                                                     _stream(x.device))
    _lib.check(code, "stp3_upsample2x_window_f32")
    return y


def upsample2x_backward_from(gy: torch.Tensor, coff: int, C: int) -> torch.Tensor:
    """Adjoint of upsample2x applied to channels [coff, coff + C) of gy (N, 2h, 2w, Cy) -> dense (N, h, w, C)."""
    _f32_cl(gy)
    N, H2, W2, Cy = gy.shape
    assert H2 % 2 == 0 and W2 % 2 == 0 and 0 <= coff and coff + C <= Cy
    gx = torch.empty((N, H2 // 2, W2 // 2, C), dtype=torch.float32, device=gy.device)
    with torch.cuda.device(gy.device):
        code = _lib.lib().stp3_upsample2x_window_bwd(gy.data_ptr(), Cy, coff, N, H2 // 2, W2 // 2, C, gx.data_ptr(),
                                                     _stream(gy.device))
    _lib.check(code, "stp3_upsample2x_window_bwd")
    return gx


def sigmoid_backward(g: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """dL/dz of s = sigmoid(z) from g = dL/ds and the forward output s (same shape, contiguous fp32)."""
    assert g.shape == s.shape and g.is_contiguous() and s.is_contiguous()
    dz = torch.empty_like(s)
    with torch.cuda.device(s.device):
        code = _lib.lib().stp3_sigmoid_bwd(g.data_ptr(), s.data_ptr(), s.numel(), dz.data_ptr(), _stream(s.device))
    _lib.check(code, "stp3_sigmoid_bwd")
    return dz



# ------------------------------------------------------------------------------------------------ EfficientNet trunk
# Train mode of the native trunk (models/efficientnet.py, include/stp3_b200.h "EfficientNet trunk, train mode").
def conv1x1_raw(x: dense.HL, weight: torch.Tensor) -> torch.Tensor:
    """conv_raw of a 1x1 convolution with any number of output channels: more than 256 (the trunk's expand
    convolutions) run as column chunks of at most 256 whose fp32 outputs are concatenated."""
    cout = weight.shape[0]
    if cout <= 256:
        return conv_raw(x, weight, 1)
    return torch.cat([conv_raw(x, weight[n0:n0 + 256], 1) for n0 in range(0, cout, 256)], dim=-1)


def conv1x1_dgrad(g: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """conv_dgrad of a 1x1 convolution with any number of input channels (the trunk's projections): g is converted to
    hi/lo once, and more than 256 input channels run as chunks whose fp32 outputs are concatenated."""
    _f32_cl(g)
    N, H, W, _ = g.shape
    cin = weight.shape[1]
    g_hl = to_hl(g)
    outs = []
    for c0 in range(0, cin, 256):
        w = weight[:, c0:c0 + 256]
        out = torch.empty((N, H, W, w.shape[1]), dtype=torch.float32, device=g.device)
        dense.conv(g_hl, pack_dgrad(w, 1, 0)[0][1], out_f32=out, n_valid=w.shape[1], out_f32_nhwc=True, store=False,
                   tune=(0, 0))
        outs.append(out)
    return outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)


def stem_raw(x: torch.Tensor, weight: torch.Tensor, out_hw: Tuple[int, int], pad: int) -> torch.Tensor:
    """x (M, 3, H, W) fp32 NCHW images -> (M, Ho, Wo, cout) fp32: the 3x3 stride-2 stem convolution, no BatchNorm, no
    activation (stp3_effnet_stem_raw); pad = the top / left static pad."""
    assert x.dtype == torch.float32 and x.is_contiguous() and x.is_cuda and x.dim() == 4 and x.shape[1] == 3
    M, _, H, W = x.shape
    cout = weight.shape[0]
    w = weight.detach().float().contiguous()
    y = torch.empty((M, *out_hw, cout), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_effnet_stem_raw(x.data_ptr(), M, H, W, out_hw[0], out_hw[1], pad, pad, w.data_ptr(), cout,
                                               y.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_effnet_stem_raw")
    return y


def stem_wgrad(x: torch.Tensor, g: torch.Tensor, pad: int) -> torch.Tensor:
    """dL/dW (cout, 3, 3, 3) of stem_raw from its images x and g = dL/dy (M, Ho, Wo, cout) (stp3_effnet_stem_wgrad)."""
    _f32_cl(g)
    M, _, H, W = x.shape
    _, Ho, Wo, cout = g.shape
    L = _lib.lib()
    nbytes = L.stp3_effnet_stem_wgrad_scratch_bytes(M, Ho, Wo, cout)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    dw = torch.empty((cout, 3, 3, 3), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = L.stp3_effnet_stem_wgrad(x.data_ptr(), M, H, W, Ho, Wo, pad, pad, g.data_ptr(), cout, dw.data_ptr(),
                                        scratch.data_ptr(), nbytes, _stream(x.device))
    _lib.check(code, "stp3_effnet_stem_wgrad")
    return dw


def _dw_desc(N: int, H: int, W: int, Ho: int, Wo: int, k: int, stride: int, pad: int, C: int):
    return _lib.DwDesc(n_img=N, H=H, W=W, Ho=Ho, Wo=Wo, k=k, stride=stride, pad_t=pad, pad_l=pad, C=C, in_cstride=C,
                       out_cstride=C)


def _dw_taps(weight: torch.Tensor) -> torch.Tensor:
    """depthwise weight (C, 1, k, k) -> the kernels' [k*k][C] layout"""
    C, k = weight.shape[0], weight.shape[-1]
    return weight.detach().float().reshape(C, k * k).t().contiguous()


def dw_raw(x: torch.Tensor, weight: torch.Tensor, stride: int, pad: int, out_hw: Tuple[int, int]) -> torch.Tensor:
    """Depthwise convolution of x (N, H, W, C) with weight (C, 1, k, k), top / left pad `pad`, zero past the bottom /
    right edge -> (N, Ho, Wo, C) fp32, no BatchNorm, no activation (stp3_dw_fwd_raw)."""
    _f32_cl(x)
    N, H, W, C = x.shape
    k = weight.shape[-1]
    d = _dw_desc(N, H, W, *out_hw, k, stride, pad, C)
    w = _dw_taps(weight)
    y = torch.empty((N, *out_hw, C), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_dw_fwd_raw(ctypes.byref(d), x.data_ptr(), w.data_ptr(), y.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_dw_fwd_raw")
    return y


def dw_dgrad(g: torch.Tensor, weight: torch.Tensor, stride: int, pad: int, in_hw: Tuple[int, int]) -> torch.Tensor:
    """dL/dx (N, H, W, C) of dw_raw from g = dL/dy (N, Ho, Wo, C): its exact adjoint (stp3_dw_dgrad)."""
    _f32_cl(g)
    N, Ho, Wo, C = g.shape
    k = weight.shape[-1]
    d = _dw_desc(N, *in_hw, Ho, Wo, k, stride, pad, C)
    w = _dw_taps(weight)
    dx = torch.empty((N, *in_hw, C), dtype=torch.float32, device=g.device)
    with torch.cuda.device(g.device):
        code = _lib.lib().stp3_dw_dgrad(ctypes.byref(d), g.data_ptr(), w.data_ptr(), dx.data_ptr(), _stream(g.device))
    _lib.check(code, "stp3_dw_dgrad")
    return dx


def dw_wgrad(x: torch.Tensor, g: torch.Tensor, k: int, stride: int, pad: int) -> torch.Tensor:
    """dL/dW (C, 1, k, k) of dw_raw from its input x (N, H, W, C) and g = dL/dy (N, Ho, Wo, C) (stp3_dw_wgrad)."""
    _f32_cl(x), _f32_cl(g)
    N, H, W, C = x.shape
    _, Ho, Wo, _ = g.shape
    d = _dw_desc(N, H, W, Ho, Wo, k, stride, pad, C)
    L = _lib.lib()
    nbytes = L.stp3_dw_wgrad_scratch_bytes(ctypes.byref(d))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    dw = torch.empty((k * k, C), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        code = L.stp3_dw_wgrad(ctypes.byref(d), x.data_ptr(), g.data_ptr(), dw.data_ptr(), scratch.data_ptr(), nbytes,
                               _stream(x.device))
    _lib.check(code, "stp3_dw_wgrad")
    return dw.t().reshape(C, 1, k, k).contiguous()


def _bn_vectors(st: Optional[BNStats], bn: Optional[nn.Module]):
    if st is None:
        return None, None, None, None
    return st.mean, st.invstd, bn.weight.detach().float().contiguous(), bn.bias.detach().float().contiguous()


def bn_act(x: torch.Tensor, st: Optional[BNStats], bn: Optional[nn.Module], swish: bool,
           mul: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
           hl: bool = False, f32: bool = True) -> Tuple[Optional[torch.Tensor], Optional[dense.HL]]:
    """y = act(BN(x)) * mul[img] * scale[img] + res on x (N, H, W, C) (stp3_trunk_bn_act): BN with the batch statistics
    st and bn's gamma / beta (st None: no BatchNorm), act swish or the identity, mul (N, C) (the squeeze-excite gate),
    scale (N,) (drop-connect), res (N, H, W, C) (identity skip) -> (fp32 y or None, hi/lo planes or None)."""
    _f32_cl(x)
    N, H, W, C = x.shape
    dev = x.device
    for t in (mul, scale):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() in (N, N * C))
    if res is not None:
        _f32_cl(res)
        assert res.shape == x.shape
    y = torch.empty_like(x) if f32 else None
    out = dense.HL.empty(N, 1, H, W, C, dev) if hl else None
    mean, invstd, gam, bet = _bn_vectors(st, bn)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_trunk_bn_act(x.data_ptr(), N * H * W, C, H * W, _p(mean), _p(invstd), _p(gam), _p(bet),
                                            int(swish), _p(mul), _p(scale), _p(res), _p(y),
                                            _p(out.hi if out else None), _p(out.lo if out else None),
                                            out.hi.shape[-1] if out else 0, _stream(dev))
    _lib.check(code, "stp3_trunk_bn_act")
    return y, out


def bn_act_grad(g: torch.Tensor, x: Optional[torch.Tensor], st: Optional[BNStats], bn: Optional[nn.Module],
                swish: bool, mul: Optional[torch.Tensor] = None, add: Optional[torch.Tensor] = None,
                scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dL/dz = (g * mul[img] + add[img]) * act'(z) * scale[img], z = BN(x) recomputed from x and st
    (stp3_trunk_bn_act_bwd): what bn_backward then takes, with no ReLU mask."""
    _f32_cl(g)
    N, H, W, C = g.shape
    if x is not None:
        assert x.shape == g.shape and x.is_contiguous()
    mean, invstd, gam, bet = _bn_vectors(st, bn)
    out = torch.empty_like(g)
    with torch.cuda.device(g.device):
        code = _lib.lib().stp3_trunk_bn_act_bwd(g.data_ptr(), _p(x), N * H * W, C, H * W, _p(mean), _p(invstd),
                                                _p(gam), _p(bet), int(swish), _p(mul), _p(add), _p(scale),
                                                out.data_ptr(), _stream(g.device))
    _lib.check(code, "stp3_trunk_bn_act_bwd")
    return out


def image_channel_dot(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """(N, C) fp32: per image and channel, the sum over pixels of a * b (a, b (N, H, W, C)) in a fixed order
    (stp3_image_channel_dot)."""
    _f32_cl(a), _f32_cl(b)
    assert a.shape == b.shape
    N, H, W, C = a.shape
    L = _lib.lib()
    nbytes = L.stp3_image_channel_dot_scratch_bytes(N, H * W, C)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=a.device)
    out = torch.empty((N, C), dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        code = L.stp3_image_channel_dot(a.data_ptr(), b.data_ptr(), N, H * W, C, out.data_ptr(), scratch.data_ptr(),
                                        nbytes, _stream(a.device))
    _lib.check(code, "stp3_image_channel_dot")
    return out


def se_backward(dgate: torch.Tensor, gate: torch.Tensor, sums: torch.Tensor, hw: int, w_r: torch.Tensor,
                b_r: torch.Tensor, w_e: torch.Tensor):
    """The squeeze-excite chain backward of every image (stp3_se_bwd): from dL/dgate, the forward's gate and spatial
    sums (N, C) and the weights w_r (R, C), b_r (R), w_e (C, R) -> (de (N, C), swish(r) (N, R), dr (N, R),
    dL/dmean / hw (N, C))."""
    N, C = gate.shape
    R = w_r.shape[0]
    for t in (dgate, gate, sums, w_r, b_r, w_e):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert dgate.shape == sums.shape == (N, C) and w_r.shape == (R, C) and w_e.shape == (C, R) and b_r.numel() == R
    de, dmean = (torch.empty((N, C), dtype=torch.float32, device=gate.device) for _ in range(2))
    sr, dr = (torch.empty((N, R), dtype=torch.float32, device=gate.device) for _ in range(2))
    with torch.cuda.device(gate.device):
        code = _lib.lib().stp3_se_bwd(dgate.data_ptr(), gate.data_ptr(), sums.data_ptr(), N, C, 1.0 / hw,
                                      w_r.data_ptr(), b_r.data_ptr(), R, w_e.data_ptr(), de.data_ptr(), sr.data_ptr(),
                                      dr.data_ptr(), dmean.data_ptr(), _stream(gate.device))
    _lib.check(code, "stp3_se_bwd")
    return de, sr, dr, dmean
