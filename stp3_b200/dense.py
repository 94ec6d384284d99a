"""Host side of the dense (tensor-core) path: activation container, weight folding/packing, conv launcher.

Activations live on the device channels-last as two bf16 planes (hi, lo) with channels padded to a multiple of 64;
weights are folded (eval-mode BatchNorm -> scale/shift, reference: nn.BatchNorm eps 1e-5) and packed once per
checkpoint load into the tap-major / K-major layout stp3_conv_fwd expects (include/stp3_b200.h).
"""
import ctypes
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib

KB = 64  # channels per K block


def pad_to(c: int, m: int = KB) -> int:
    return (c + m - 1) // m * m


def out_tile(c: int) -> int:
    """Padded output-channel tile of the conv kernel (UMMA N): 64, 128 or 256."""
    for bn in (64, 128, 256):
        if c <= bn:
            return bn
    raise ValueError(f"{c} output channels: split the convolution (max 256 per launch)")


@dataclass
class HL:
    """(B, T, H, W, Cp) fp32 tensor carried as bf16 hi/lo planes; `c` = number of real channels.  lo None: ONE 16-bit
    plane (hi.dtype torch.bfloat16 or torch.float16), the operand of the autocast train path (dense_train)."""
    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    c: int

    @property
    def shape(self):
        return self.hi.shape

    @staticmethod
    def empty(B, T, H, W, c, device, cp=None):
        cp = cp or pad_to(c)
        return HL(torch.empty((B, T, H, W, cp), dtype=torch.bfloat16, device=device),
                  torch.empty((B, T, H, W, cp), dtype=torch.bfloat16, device=device), c)

    @staticmethod
    def zeros(B, T, H, W, c, device, cp=None):
        cp = cp or pad_to(c)
        return HL(torch.zeros((B, T, H, W, cp), dtype=torch.bfloat16, device=device),
                  torch.zeros((B, T, H, W, cp), dtype=torch.bfloat16, device=device), c)


def split_hilo(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def fold_bn(weight: torch.Tensor, bn: Optional[torch.nn.modules.batchnorm._BatchNorm], conv_bias=None):
    """conv (no bias) -> eval BatchNorm  ==  conv with w*s and bias (beta - mean*s), s = gamma/sqrt(var+eps)."""
    cout = weight.shape[0]
    w = weight.detach().float()
    b = conv_bias.detach().float() if conv_bias is not None else torch.zeros(cout, device=w.device)
    if bn is not None:
        s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
        w = w * s.view(-1, *([1] * (w.dim() - 1)))
        b = (b - bn.running_mean.detach().float()) * s + bn.bias.detach().float()
    return w, b


@dataclass
class PackedConv:
    w: torch.Tensor            # [ntaps][cin_p/64][2][bn][64] bf16
    bias: torch.Tensor         # [bn] fp32
    taps: List[Tuple[int, int, int]]
    cin_p: int
    bn: int
    cout: int
    stride: int
    k_lo: int = 0              # input channels [k_lo, k_hi) of the window carry weights (multiples of 16)
    k_hi: int = 0
    uid: int = 0               # identity of this packing for the autotune cache (a data_ptr can be reused after a repack)
    plane: Optional[torch.dtype] = None   # None: w holds hi/lo planes; torch.bfloat16 / torch.float16: w is
                                          # [ntaps][cin_p/64][bn][64] of that type (stp3_conv_fwd_plane)


PLANE_OPERAND = {torch.bfloat16: _lib.OPERAND_BF16, torch.float16: _lib.OPERAND_F16}


def pack_planes(m: torch.Tensor, plane: Optional[torch.dtype] = None) -> torch.Tensor:
    """Tap matrices m (ntaps, bn, cin_p) fp32 -> the weight operand of stp3_conv_fwd: [tap][K block][hi, lo][bn][64] bf16,
    or with plane (torch.bfloat16 / torch.float16) one plane [tap][K block][bn][64] of m rounded to that type."""
    nt, bn, cin_p = m.shape
    kbs = cin_p // KB
    if plane is not None:
        return m.to(plane).view(nt, bn, kbs, KB).permute(0, 2, 1, 3).contiguous()
    hi, lo = split_hilo(m)
    packed = torch.stack([hi.view(nt, bn, kbs, KB), lo.view(nt, bn, kbs, KB)], dim=0)   # (2, nt, bn, kbs, 64)
    return packed.permute(1, 3, 0, 2, 4).contiguous()                                   # (nt, kbs, 2, bn, 64)


_PACK_COUNTER = 0


def pack_conv(weight: torch.Tensor, bias: torch.Tensor, *, stride: int = 1, dilation: int = 1,
              padding: Optional[int] = None, causal_time: bool = True, cin_p: Optional[int] = None,
              bn: Optional[int] = None, prune_extent: Optional[Tuple[int, int]] = None,
              in_layout: Optional[Sequence[Tuple[int, int, int]]] = None,
              plane: Optional[torch.dtype] = None) -> PackedConv:
    """weight: (Cout, Cin, kh, kw) or (Cout, Cin, kt, kh, kw), already BN-folded; bias (Cout).
    Taps are (dt, dy, dx) input offsets: dy = ky*dilation - padding (padding defaults to 'same'); for 3-D kernels
    dt = kt_index - (kt - 1) (causal: the reference pads time on the left only, temporal.py:256-262).
    plane (torch.bfloat16 / torch.float16): one plane of the weights rounded to that type (pack_planes)."""
    if weight.dim() == 4:
        weight = weight.unsqueeze(2)
    cout, cin, kt, kh, kw = weight.shape
    pad_h = padding if padding is not None else (kh - 1) * dilation // 2
    pad_w = padding if padding is not None else (kw - 1) * dilation // 2
    # in_layout: [(first logical input channel, count, physical channel offset)] -- where each group of the
    # convolution's input channels lives inside the (padded / concatenated) physical input window
    in_layout = list(in_layout) if in_layout is not None else [(0, cin, 0)]
    cin_p = cin_p or pad_to(max(off + n for _, n, off in in_layout))
    bn = bn or out_tile(cout)
    dev = weight.device
    taps, mats = [], []
    for it in range(kt):
        for ix in range(kw):              # dy innermost: runs of taps whose dy advance by the stride share one
            # activation load (stride 1: dy, dy+1, dy+2; stride 2: the even rows of the kernel, then the odd ones)
            for iy in (list(range(0, kh, 2)) + list(range(1, kh, 2)) if stride == 2 else range(kh)):
                dy, dx = iy * dilation - pad_h, ix * dilation - pad_w
                if prune_extent is not None and stride == 1:
                    # a tap whose shift exceeds the image reads only zero padding for every output pixel
                    H, W = prune_extent
                    if abs(dy) >= H or abs(dx) >= W:
                        continue
                taps.append((it - (kt - 1) if causal_time else it, dy, dx))
                m = torch.zeros((bn, cin_p), dtype=torch.float32, device=dev)
                for src, n, off in in_layout:
                    m[:cout, off:off + n] = weight[:, src:src + n, it, iy, ix]
                mats.append(m)
    packed = pack_planes(torch.stack(mats), plane)                   # mats: (ntaps, bn, cin_p)
    b = torch.zeros(bn, dtype=torch.float32, device=dev)
    b[:cout] = bias
    k_lo = min(off for _, _, off in in_layout) // 16 * 16
    k_hi = (max(off + n for _, n, off in in_layout) + 15) // 16 * 16
    if not (k_lo < KB and k_hi > cin_p - KB):          # the kernel trims only the first / last 64-channel block
        k_lo, k_hi = 0, cin_p
    global _PACK_COUNTER
    _PACK_COUNTER += 1
    return PackedConv(packed, b, taps, cin_p, bn, cout, stride, k_lo, k_hi, _PACK_COUNTER, plane)


# ------------------------------------------------------------------------------------------------ autotuner
# The conv kernel has tiling knobs (sharing one activation load between the dy taps of a 3x3, streaming the weights
# through the ring instead of keeping them resident, the stacked hi/lo weight operand, 64-column blocks for layers of
# 128 / 256 columns).  Which combination wins depends on the layer (K depth, N width, image size, whether the weights
# are smem-resident), so the first eager call of every (layer, shape) times the candidates back to back and the winner
# is cached; CUDA-graph capture then records the tuned launches.  STP3_CONV_AUTOTUNE=0 disables it (kernel heuristics,
# and untuned_blocks() for the column blocks).  So does torch.use_deterministic_algorithms: tilings do not all give the
# same bits, and one picked by timing can differ between processes.  The mode is part of the cache key, so a tiling
# timed with the flag off is never reused with it on.
import os as _os

_TUNED = {}
_AUTOTUNE = _os.environ.get("STP3_CONV_AUTOTUNE", "1") != "0"
TUNE_LOG = []      # (description, {config: ms}) for reports


BLOCKS64 = 16      # bit of a tiling's group: 64-column blocks (stp3_conv_desc.tune_bn = 64)


def tune_candidates(pc: PackedConv, per_image: bool = False) -> List[Tuple[int, int]]:
    """The (n_sub, group) tilings the autotuner times for this packed convolution.  Per-image weights are never
    resident: only the streamed (+4) tilings are offered for them.  Convolutions of 128 / 256 columns are also offered
    in 64-column blocks (+16), plain and with the stacked operand (+8); their weights stream either way."""
    taps = pc.taps
    groupable = any(taps[i + 1][0] == taps[i][0] and taps[i + 1][2] == taps[i][2] and
                    taps[i + 1][1] == taps[i][1] + pc.stride for i in range(len(taps) - 1))
    cands = [(1, 1)] + ([(1, 3)] if groupable else [])
    if per_image:
        cands = [(ns, g + 4) for ns, g in cands]
    elif len(taps) > 1:   # weights streamed through the ring instead of resident: more activation stages in flight
        cands += [(ns, g + 4) for ns, g in cands]
    if pc.bn == 64:     # stacked [W_hi; W_lo] operand: two MMAs per product instead of three
        cands += [(ns, g + 8) for ns, g in cands]
    else:
        cands += [(1, g + (4 if per_image else 0) + BLOCKS64 + s) for s in (8, 0) for g in sorted({g & 3 for _, g in cands})]
    return cands


def untuned_blocks(pc: PackedConv, tiles: int, n_sm: int) -> int:
    """The group bits of the column blocks when nothing was timed: 64-column stacked blocks where 128-column items
    would not fill two waves of the SMs, else the kernel's own choice."""
    return BLOCKS64 + 8 if pc.bn >= 128 and tiles * (pc.bn // 128) < 2 * n_sm else 0


def _tune(key, desc, launch, cands):
    times = {}
    for ns, g in cands:
        launch(ns, g)                                   # warm (descriptor / attribute setup)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(4):
            launch(ns, g)
        b.record()
        b.synchronize()
        times[(ns, g)] = a.elapsed_time(b) / 4
    best = min(times, key=times.get)
    _TUNED[key] = best
    TUNE_LOG.append((desc, times))
    return best


def conv(x: HL, pc: PackedConv, *, cin_off: int = 0, out: Optional[HL] = None, out_coff: int = 0, relu: bool = False,
         img_bias: Optional[torch.Tensor] = None, residual: Optional[HL] = None, res_coff: int = 0,
         res_after_act: bool = False, out_f32: Optional[torch.Tensor] = None, n_valid: int = 0, sigmoid: bool = False,
         out_hw: Optional[Tuple[int, int]] = None, n_store: int = 0, frames: Optional[Tuple[int, int]] = None,
         head: Optional[dict] = None, store: bool = True, tune: Optional[Tuple[int, int]] = None,
         col_sums: Optional[torch.Tensor] = None, out2: Optional[HL] = None, out2_coff: int = 0, n_store2: int = 0,
         relu2: bool = False, out_f32_nhwc: bool = False, swish: bool = False, w_img_stride: int = 0) -> Optional[HL]:
    """y = act(conv(x[..., cin_off:cin_off+cin]) + bias [+ residual]) written into out[..., out_coff:...]; when
    img_bias (n_img, bn) is given it REPLACES the convolution's bias vector (build it with bias_table()).
    out2 (bn = 128 layers, n_store <= 64): output columns [64, 64+n_store2) go to out2[..., out2_coff:...] with activation
    relu2 -- two 64-column convolutions of the same input in one launch.
    col_sums (B*T, 64) fp32 (bn = 64 layers): receives the per-image sums over pixels of the activated output.
    tune = (n_sub, group) forces a tiling (n_sub is ignored: the tile is 8x16 pixels; group +4 = streamed weights,
    +8 = stacked hi/lo weight operand, +16 = 64-column blocks) instead of the autotuned one.  A fused head and a
    second destination need all columns in one block: +16 is dropped for them.
    swish: x * sigmoid(x) instead of ReLU.  w_img_stride > 0: pc.w holds image 0's weights and image i's start
    w_img_stride bf16 elements further (squeeze-excite gated projections, se_gate())."""
    B, T_total, H, W, cs = x.hi.shape
    t0, T = frames if frames is not None else (0, T_total)      # process frames [t0, t0+T) of every sample
    Ho, Wo = out_hw if out_hw is not None else ((H + pc.stride - 1) // pc.stride, (W + pc.stride - 1) // pc.stride)
    d = _lib.ConvDesc()
    d.B, d.T, d.H, d.W = B, T, H, W
    d.T_total, d.t0 = T_total, t0
    d.in_cstride, d.cin_off, d.cin = cs, cin_off, pc.cin_p
    d.Ho, d.Wo, d.stride = Ho, Wo, pc.stride
    d.ntaps = len(pc.taps)
    for i, (dt, dy, dx) in enumerate(pc.taps):
        d.taps[i][0], d.taps[i][1], d.taps[i][2] = dt, dy, dx
    d.bn = pc.bn
    d.n_cols = pc.cout              # weight rows / bias entries beyond cout are zero padding
    d.k_lo, d.k_hi = pc.k_lo, pc.k_hi
    if out is None and out_f32 is None and store:
        out = HL.empty(B, T, Ho, Wo, pc.cout, x.hi.device, cp=pc.bn)
    hd = None
    if head is not None:
        # fused 1x1 head: dict(w (KO,bn) f32, b (KO) f32, outs=[(tensor (n_img,k,Ho,Wo) f32, channel)], sigmoid_mask)
        hd = _lib.ConvHead()
        hd.n_out = len(head["outs"])
        assert head["w"].shape == (hd.n_out, pc.bn) and head["w"].is_contiguous() and head["b"].numel() == hd.n_out
        hd.w, hd.b = head["w"].data_ptr(), head["b"].data_ptr()
        for k, (t, ch) in enumerate(head["outs"]):
            assert t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == B * T and t.shape[2:] == (Ho, Wo)
            hd.out[k] = t.data_ptr() + ch * Ho * Wo * 4
            hd.img_stride[k] = t.shape[1] * Ho * Wo
        hd.sigmoid_mask = int(head.get("sigmoid_mask", 0))
    if out is not None:
        assert out.hi.shape[:4] == (B, T, Ho, Wo), (out.hi.shape, (B, T, Ho, Wo))
        d.out_cstride, d.out_coff, d.n_store = out.hi.shape[-1], out_coff, n_store
    d.relu = int(relu)
    d.swish, d.w_img_stride = int(swish), int(w_img_stride)
    if residual is not None:
        d.res_mode = 2 if res_after_act else 1
        d.res_cstride, d.res_coff = residual.hi.shape[-1], res_coff
        assert residual.hi.shape[:4] == (B, T, Ho, Wo)
    d.n_valid, d.sigmoid = n_valid, int(sigmoid)
    d.f32_layout = int(out_f32_nhwc)        # out_f32 (B*T, Ho, Wo, n_valid) instead of (B*T, n_valid, Ho, Wo)
    if out2 is not None:
        assert pc.bn == 128 and out is not None and out2.hi.shape[:4] == (B, T, Ho, Wo)
        d.y2_hi, d.y2_lo = out2.hi.data_ptr(), out2.lo.data_ptr()
        d.out2_cstride, d.out2_coff, d.n_store2, d.relu2 = out2.hi.shape[-1], out2_coff, n_store2, int(relu2)
    scratch = None
    if col_sums is not None:
        assert pc.bn == 64 and col_sums.shape == (B * T, 64) and col_sums.dtype == torch.float32 and col_sums.is_contiguous()
        nbytes = _lib.lib().stp3_conv_col_sums_scratch_bytes(B * T, 64)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.hi.device)
        d.col_sums, d.col_sums_scratch, d.col_sums_scratch_bytes = col_sums.data_ptr(), scratch.data_ptr(), nbytes
    if img_bias is not None:
        assert img_bias.shape == (B * T, pc.bn) and img_bias.dtype == torch.float32 and img_bias.is_contiguous()
    operand = PLANE_OPERAND[x.hi.dtype] if x.lo is None else _lib.OPERAND_HILO
    if operand != _lib.OPERAND_HILO:      # one-plane operands: fp32 output only (stp3_conv_fwd_plane)
        assert pc.plane == x.hi.dtype, (pc.plane, x.hi.dtype)
        assert out_f32 is not None and out is None and out2 is None and residual is None and hd is None and \
            scratch is None and not swish and not w_img_stride
    else:
        assert pc.plane is None, "one-plane weights need a one-plane input"
    dev = x.hi.device
    ptr = lambda t: t.data_ptr() if t is not None else None

    one_block = hd is not None or out2 is not None

    def launch(n_sub=0, group=0):
        d.tune_n_sub, d.tune_group = n_sub, group & ~BLOCKS64
        d.tune_bn = 64 if group & BLOCKS64 and not one_block else 0
        with torch.cuda.device(dev):
            if operand != _lib.OPERAND_HILO:
                code = _lib.lib().stp3_conv_fwd_plane(
                    ctypes.byref(d), operand, x.hi.data_ptr(), pc.w.data_ptr(), pc.bias.data_ptr(), ptr(img_bias),
                    out_f32.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
                _lib.check(code, "stp3_conv_fwd_plane")
                return
            code = _lib.lib().stp3_conv_fwd(
                ctypes.byref(d), x.hi.data_ptr(), x.lo.data_ptr(), pc.w.data_ptr(), pc.bias.data_ptr(), ptr(img_bias),
                ptr(residual.hi if residual is not None else None), ptr(residual.lo if residual is not None else None),
                ptr(out.hi if out is not None else None), ptr(out.lo if out is not None else None), ptr(out_f32),
                ctypes.byref(hd) if hd is not None else None, torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(code, "stp3_conv_fwd")

    det = torch.are_deterministic_algorithms_enabled()
    key = (pc.uid, B, T, H, W, cs, cin_off, Ho, Wo, t0, int(relu), residual is not None, out_f32 is not None,
           hd is not None, out2 is not None, int(swish), int(w_img_stride), det)
    cfg = tune if tune is not None else _TUNED.get(key)
    autotune = _AUTOTUNE and not det
    if cfg is None and autotune and not torch.cuda.is_current_stream_capturing():
        desc = f"{len(pc.taps)}tap cin{pc.cin_p} bn{pc.bn} s{pc.stride} {B * T}x{Ho}x{Wo}"
        # the tuner launches the layer many times: an output that aliases an input would be corrupted silently
        ins = {x.hi.data_ptr()} | ({x.lo.data_ptr()} if x.lo is not None else set()) | ({residual.hi.data_ptr(), residual.lo.data_ptr()} if residual is not None else set())
        outs = {t.data_ptr() for t in ((out.hi, out.lo) if out is not None else ()) + ((out2.hi, out2.lo) if out2 is not None else ())}
        assert not (ins & outs), "stp3_b200.dense.conv: output aliases an input (in-place convolution is not supported)"
        cfg = _tune(key, desc, launch, [c for c in tune_candidates(pc, per_image=w_img_stride > 0)
                                        if not (one_block and c[1] & BLOCKS64)])
    elif cfg is None and not autotune and not one_block and pc.bn >= 128:
        tiles = B * T * -(-Ho // 8) * -(-Wo // 16)
        cfg = _TUNED[key] = (0, untuned_blocks(pc, tiles, torch.cuda.get_device_properties(dev).multi_processor_count))
        TUNE_LOG.append((f"{len(pc.taps)}tap cin{pc.cin_p} bn{pc.bn} s{pc.stride} {B * T}x{Ho}x{Wo}", {cfg: float("nan")}))
    launch(*(cfg or (0, 0)))
    return out


@dataclass
class PackedAspp:
    w: torch.Tensor            # bf16 rows of 64: [tap/K blocks ...][projection blocks ...], each [hi 128][lo 128]
    br_bias: torch.Tensor      # (n_br, 128) fp32
    proj_bias: torch.Tensor    # (128,) fp32
    taps: List[List[Tuple[int, int]]]
    cin_p: int


def pack_aspp(branches, proj_w: torch.Tensor, proj_b: torch.Tensor) -> PackedAspp:
    """branches: [(weight (128, Cin, kh, kw) BN-folded, bias (128), dilation)]; proj_w (<= 128, n_br * 128) BN-folded
    (fewer than 128 output rows are zero-padded).  Layout of stp3_aspp_fused_fwd (include/stp3_b200.h)."""
    h = 128
    if proj_w.shape[0] < h:
        pw = torch.zeros((h, proj_w.shape[1]), dtype=proj_w.dtype, device=proj_w.device)
        pw[:proj_w.shape[0]] = proj_w
        pb = torch.zeros(h, dtype=proj_b.dtype, device=proj_b.device)
        pb[:proj_b.shape[0]] = proj_b
        proj_w, proj_b = pw, pb
    cin = branches[0][0].shape[1]
    cin_p = pad_to(cin)
    kbs = cin_p // KB
    dev = proj_w.device
    blocks, taps_all, biases = [], [], []
    for w, b, dil in branches:
        assert w.shape[0] == h and w.shape[1] == cin
        kh, kw = w.shape[2:]
        taps = []
        for iy in range(kh):
            for ix in range(kw):
                dy, dx = (iy - (kh - 1) // 2) * dil, (ix - (kw - 1) // 2) * dil
                taps.append((dy, dx))
                m = torch.zeros((h, cin_p), dtype=torch.float32, device=dev)
                m[:, :cin] = w[:, :, iy, ix]
                for kb in range(kbs):
                    blocks.append(m[:, kb * KB:(kb + 1) * KB])
        taps_all.append(taps)
        biases.append(b)
    for i in range(len(branches)):
        for kb2 in range(2):
            blocks.append(proj_w[:, i * h + kb2 * KB: i * h + (kb2 + 1) * KB])
    m = torch.stack(blocks).float()                                   # (n_blocks, 128, 64)
    hi, lo = split_hilo(m)
    packed = torch.stack([hi, lo], dim=1).contiguous()                # (n_blocks, 2, 128, 64)
    return PackedAspp(packed, torch.stack(biases).float().contiguous(), proj_b.float().contiguous(), taps_all, cin_p)


def aspp_fused(x: HL, pa: PackedAspp, img_bias: torch.Tensor, out: Optional[HL] = None, out_coff: int = 0,
               relu: bool = True, n_store: int = 128, c_out: Optional[int] = None) -> HL:
    """y = [relu](project(cat_b relu(branch_b(x))) + img_bias): stp3_aspp_fused_fwd.  n_store = 64: only the first 64
    output channels exist (c_out of them real)."""
    B, T, H, W, cs = x.hi.shape
    if out is None:
        out = HL.empty(B, T, H, W, c_out or n_store, x.hi.device, cp=n_store)
    assert img_bias.shape == (B * T, 128) and img_bias.dtype == torch.float32 and img_bias.is_contiguous()
    d = _lib.AsppDesc()
    d.B, d.T, d.H, d.W, d.in_cstride, d.cin = B, T, H, W, cs, pa.cin_p
    d.n_br = len(pa.taps)
    for b, taps in enumerate(pa.taps):
        d.n_taps[b] = len(taps)
        for i, (dy, dx) in enumerate(taps):
            d.taps[b][i][0], d.taps[b][i][1] = dy, dx
    d.out_cstride, d.out_coff = out.hi.shape[-1], out_coff
    d.no_relu, d.n_store = int(not relu), n_store
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_aspp_fused_fwd(ctypes.byref(d), x.hi.data_ptr(), x.lo.data_ptr(), pa.w.data_ptr(),
                                              pa.br_bias.data_ptr(), img_bias.data_ptr(), out.hi.data_ptr(),
                                              out.lo.data_ptr(), torch.cuda.current_stream(x.hi.device).cuda_stream)
    _lib.check(code, "stp3_aspp_fused_fwd")
    return out


@dataclass
class PackedBlockTail:
    w: torch.Tensor                 # (n_blocks, 2, 128, 64) bf16
    chains: list                    # [(src, cin_off, taps [(dt,dy,dx)], n_mma, tmem_col, k_lo, k_hi)]
    res: Optional[tuple]            # the projection chain or None (identity residual)
    piece_col: List[int]


def _pair_rows(m: torch.Tensor) -> torch.Tensor:
    """(N, 64) weight rows of an N-wide chain -> (128, 64): row n of the first / second half of N at row n / 64 + n - N/2
    (each CTA of a pair loads 64 rows and multiplies its N/2)."""
    n = m.shape[0]
    out = torch.zeros((128, KB), dtype=torch.float32, device=m.device)
    out[:n // 2] = m[:n // 2]
    out[64:64 + n - n // 2] = m[n // 2:]
    return out


def pack_block_tail(chains, agg_w: torch.Tensor, res_w: Optional[torch.Tensor], piece_col) -> PackedBlockTail:
    """chains: [(src, cin_off, weight (cout, cin, kt, kh, kw) BN-folded, k_off, n_mma, tmem_col)] -- cin input channels of
    the chain sit at channels [k_off, k_off + cin) of its 64-channel K block; agg_w (64, 128) aggregation weights in P
    order; res_w (64, cs) projection weights or None."""
    dev = agg_w.device
    blocks, desc = [], []
    for src, cin_off, w, k_off, n_mma, tmem_col in chains:
        cout, cin, kt, kh, kw = w.shape
        assert cout <= n_mma and k_off + cin <= KB
        taps = []
        for it in range(kt):
            for ix in range(kw):
                for iy in range(kh):
                    taps.append((it - (kt - 1), iy - (kh - 1) // 2, ix - (kw - 1) // 2))
                    m = torch.zeros((n_mma, KB), dtype=torch.float32, device=dev)
                    m[:cout, k_off:k_off + cin] = w[:, :, it, iy, ix]
                    blocks.append(_pair_rows(m))
        desc.append((src, cin_off, taps, n_mma, tmem_col, k_off // 16 * 16, (k_off + cin + 15) // 16 * 16))
    for kb2 in range(2):
        blocks.append(_pair_rows(agg_w[:, kb2 * KB:(kb2 + 1) * KB].float()))
    res = None
    if res_w is not None:
        cs = res_w.shape[1]
        m = torch.zeros((64, KB), dtype=torch.float32, device=dev)
        m[:res_w.shape[0], :cs] = res_w
        blocks.append(_pair_rows(m))
        res = (1, 0, [(0, 0, 0)], 64, 0, 0, (cs + 15) // 16 * 16)
    hi, lo = split_hilo(torch.stack(blocks))
    return PackedBlockTail(torch.stack([hi, lo], dim=1).contiguous(), desc, res, list(piece_col))


def block_tail(mid: HL, x: HL, pb: PackedBlockTail, hid_bias: torch.Tensor, img_bias: torch.Tensor,
               res_bias: Optional[torch.Tensor], col_sums: Optional[torch.Tensor] = None) -> HL:
    """stp3_block_fused_fwd: the paths, the aggregation convolution and the residual of a TemporalBlock in one kernel."""
    B, T, H, W, _ = x.hi.shape
    out = HL.empty(B, T, H, W, 64, x.hi.device, cp=64)
    d = _lib.BlockDesc()
    d.B, d.T, d.H, d.W = B, T, H, W
    d.mid_cstride, d.x_cstride, d.out_cstride = mid.hi.shape[-1], x.hi.shape[-1], 64

    def fill(dst, c):
        src, cin_off, taps, n_mma, tmem_col, k_lo, k_hi = c
        dst.src, dst.cin_off, dst.n_taps, dst.n_mma, dst.tmem_col, dst.k_lo, dst.k_hi = src, cin_off, len(taps), n_mma, tmem_col, k_lo, k_hi
        for i, (dt, dy, dx) in enumerate(taps):
            dst.taps[i][0], dst.taps[i][1], dst.taps[i][2] = dt, dy, dx
    d.n_chain = len(pb.chains)
    for i, c in enumerate(pb.chains):
        fill(d.chain[i], c)
    d.has_res_proj = int(pb.res is not None)
    if pb.res is not None:
        fill(d.res, pb.res)
    for i, v in enumerate(pb.piece_col):
        d.piece_col[i] = v
    n_img = B * T
    assert hid_bias.shape == (n_img, 128) and img_bias.shape == (n_img, 64) and hid_bias.is_contiguous() and img_bias.is_contiguous()
    assert (res_bias is None) == (pb.res is None)
    scratch, nbytes = None, 0
    if col_sums is not None:
        assert col_sums.shape == (n_img, 64) and col_sums.dtype == torch.float32 and col_sums.is_contiguous()
        nbytes = _lib.lib().stp3_block_fused_scratch_bytes(n_img)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.hi.device)
    ptr = lambda t: t.data_ptr() if t is not None else None
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_block_fused_fwd(
            ctypes.byref(d), mid.hi.data_ptr(), mid.lo.data_ptr(), x.hi.data_ptr(), x.lo.data_ptr(), pb.w.data_ptr(),
            hid_bias.data_ptr(), img_bias.data_ptr(), ptr(res_bias), out.hi.data_ptr(), out.lo.data_ptr(), ptr(col_sums),
            ptr(scratch), nbytes, torch.cuda.current_stream(x.hi.device).cuda_stream)
    _lib.check(code, "stp3_block_fused_fwd")
    return out


def bias_table(pc: PackedConv, n_img: int) -> torch.Tensor:
    """(n_img, bn) per-image bias initialised with the convolution's own bias; the spatially constant branches are
    accumulated on top (pool_bias / small_linear with accumulate=True)."""
    return pc.bias.unsqueeze(0).expand(n_img, -1).contiguous()


# ------------------------------------------------------------------------------------------------ aux kernels
def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def from_f32(x: torch.Tensor, channels_last: bool = False, cp: Optional[int] = None) -> HL:
    """x (B,T,C,H,W) [or (B,T,H,W,C)] fp32 on the device -> HL (CUDA transpose + hi/lo split)."""
    if not x.is_cuda:
        raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
    x = x.detach().float().contiguous()
    if channels_last:
        B, T, H, W, C = x.shape
    else:
        B, T, C, H, W = x.shape
    out = HL.empty(B, T, H, W, C, x.device, cp=cp)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_f32_to_hilo(x.data_ptr(), int(channels_last), B * T, C, H, W, out.hi.shape[-1],
                                           out.hi.data_ptr(), out.lo.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_f32_to_hilo")
    return out


def to_f32(x: HL, c_off: int = 0, c: Optional[int] = None) -> torch.Tensor:
    """HL -> (B,T,C,H,W) fp32 (the reference's layout)."""
    B, T, H, W, cs = x.hi.shape
    c = c if c is not None else x.c
    out = torch.empty((B, T, c, H, W), dtype=torch.float32, device=x.hi.device)
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_hilo_to_f32(x.hi.data_ptr(), x.lo.data_ptr(), B * T, H, W, cs, c_off, c, out.data_ptr(),
                                           _stream(x.hi.device))
    _lib.check(code, "stp3_hilo_to_f32")
    return out


def spatial_sum(x: HL) -> torch.Tensor:
    """(B*T, cstride) fp32 sums over the H*W pixels of every image.  Under torch.use_deterministic_algorithms the sums
    are added in a fixed order (stp3_spatial_sum_det) instead of with float atomics."""
    B, T, H, W, cs = x.hi.shape
    dev = x.hi.device
    out = torch.empty((B * T, cs), dtype=torch.float32, device=dev)
    L = _lib.lib()
    if torch.are_deterministic_algorithms_enabled():
        nbytes = L.stp3_spatial_sum_det_scratch_bytes(B * T, H * W, cs)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            code = L.stp3_spatial_sum_det(x.hi.data_ptr(), x.lo.data_ptr(), B * T, H * W, cs, out.data_ptr(),
                                          scratch.data_ptr(), nbytes, _stream(dev))
        _lib.check(code, "stp3_spatial_sum_det")
        return out
    with torch.cuda.device(dev):
        code = L.stp3_spatial_sum(x.hi.data_ptr(), x.lo.data_ptr(), B * T, H * W, cs, out.data_ptr(), _stream(dev))
    _lib.check(code, "stp3_spatial_sum")
    return out


def pool_bias(sums: torch.Tensor, T: int, C: int, hw: int, temporal: bool, W1, b1, W2, out: torch.Tensor,
              accumulate: bool, const: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None):
    """out[img, :CO] = (out | bias | 0) + W2 relu(W1 mean + b1): a spatially constant branch as a per-image bias (see
    header).  const (n_img, n_const): values of the trailing spatially constant input channels (not part of sums)."""
    n_img = sums.shape[0]
    R, CO = W1.shape[0], W2.shape[0]
    nc = 0 if const is None else const.shape[1]
    assert W1.shape == (R, C) and W2.shape == (CO, R) and out.shape[0] == n_img and C - nc <= sums.shape[1]
    for t in (sums, W1, b1, W2, out) + ((const,) if nc else ()) + ((bias,) if bias is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert bias is None or bias.numel() >= CO
    with torch.cuda.device(sums.device):
        code = _lib.lib().stp3_pool_bias(sums.data_ptr(), sums.shape[1], n_img, T, C, 1.0 / hw, int(temporal),
                                         const.data_ptr() if nc else None, nc,
                                         W1.data_ptr(), b1.data_ptr(), R, W2.data_ptr(), CO,
                                         bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                         out.shape[1], int(accumulate), _stream(sums.device))
    _lib.check(code, "stp3_pool_bias")


def small_linear(x: torch.Tensor, W: torch.Tensor, out: torch.Tensor, accumulate: bool,
                 bias: Optional[torch.Tensor] = None):
    """out[n, :co] = (out | bias | 0) + W x[n]."""
    n, ci = x.shape
    co = W.shape[0]
    assert W.shape == (co, ci) and out.shape[0] == n
    for t in (x, W, out) + ((bias,) if bias is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert bias is None or bias.numel() >= co
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_small_linear(x.data_ptr(), W.data_ptr(), n, ci, co,
                                            bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                            out.shape[1], int(accumulate), _stream(x.device))
    _lib.check(code, "stp3_small_linear")


def upsample2x_add(x: HL, skip: Optional[HL], c: int, skip_coff: int = 0, out: Optional[HL] = None,
                   out_coff: int = 0) -> HL:
    """out[..., out_coff:out_coff+c] = bilinear x2 (align_corners=False) of x[..., :c] (+ skip[..., skip_coff:+c])."""
    B, T, h, w, xs = x.hi.shape
    if skip is not None:
        assert skip.hi.shape[:4] == (B, T, 2 * h, 2 * w)
    if out is None:
        out = HL.empty(B, T, 2 * h, 2 * w, c, x.hi.device, cp=c)
    assert out.hi.shape[:4] == (B, T, 2 * h, 2 * w)
    ptr = lambda t: t.data_ptr() if t is not None else None
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_upsample2x_add(
            x.hi.data_ptr(), x.lo.data_ptr(), B * T, h, w, xs, ptr(skip.hi if skip else None),
            ptr(skip.lo if skip else None), skip.hi.shape[-1] if skip else 0, skip_coff, out.hi.data_ptr(),
            out.lo.data_ptr(), out.hi.shape[-1], out_coff, c, _stream(x.hi.device))
    _lib.check(code, "stp3_upsample2x_add")
    return out


# ------------------------------------------------------------------------------------------------ EfficientNet trunk
def effnet_stem(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, out_hw: Tuple[int, int], pad: Tuple[int, int],
                cp: int = KB) -> HL:
    """x (M, 3, H, W) fp32 NCHW images -> HL (M, 1, Ho, Wo, cp): 3x3 stride-2 conv (w (cout, 3, 3, 3) and b BN-folded)
    + swish; pad = (top, left) static pads."""
    if not x.is_cuda:
        raise RuntimeError("stp3_b200 dense ops run on CUDA tensors only (there is no CPU path)")
    x = x.detach().float().contiguous()
    M, C, H, W = x.shape
    assert C == 3 and w.shape[1:] == (3, 3, 3) and w.is_contiguous() and b.is_contiguous()
    Ho, Wo = out_hw
    out = HL.empty(M, 1, Ho, Wo, w.shape[0], x.device, cp=cp)
    with torch.cuda.device(x.device):
        code = _lib.lib().stp3_effnet_stem(x.data_ptr(), M, H, W, Ho, Wo, pad[0], pad[1], w.data_ptr(), b.data_ptr(),
                                           w.shape[0], cp, out.hi.data_ptr(), out.lo.data_ptr(), _stream(x.device))
    _lib.check(code, "stp3_effnet_stem")
    return out


def dw_conv(x: HL, w: torch.Tensor, b: torch.Tensor, k: int, stride: int, pad: Tuple[int, int], out_hw: Tuple[int, int],
            out: Optional[HL] = None, sums: Optional[torch.Tensor] = None) -> HL:
    """Depthwise k x k conv + folded BN + swish of channels [0, C) (w (k*k, C) fp32, b (C), C = len(b)) -> HL
    (B, T, Ho, Wo, .); sums (B*T, C) fp32 receives the per-image sums of the output (stp3_dw_fwd)."""
    B, T, H, W, cs = x.hi.shape
    C = b.numel()
    Ho, Wo = out_hw
    if out is None:
        out = HL.empty(B, T, Ho, Wo, x.c, x.hi.device, cp=pad_to(C))
    assert out.hi.shape[:4] == (B, T, Ho, Wo) and w.shape == (k * k, C) and w.is_contiguous() and b.is_contiguous()
    d = _lib.DwDesc(n_img=B * T, H=H, W=W, Ho=Ho, Wo=Wo, k=k, stride=stride, pad_t=pad[0], pad_l=pad[1], C=C,
                    in_cstride=cs, out_cstride=out.hi.shape[-1])
    scratch, nbytes = None, 0
    if sums is not None:
        assert sums.shape == (B * T, C) and sums.dtype == torch.float32 and sums.is_contiguous()
        nbytes = _lib.lib().stp3_dw_sums_scratch_bytes(ctypes.byref(d))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.hi.device)
    ptr = lambda t: t.data_ptr() if t is not None else None
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_dw_fwd(ctypes.byref(d), x.hi.data_ptr(), x.lo.data_ptr(), w.data_ptr(), b.data_ptr(),
                                      out.hi.data_ptr(), out.lo.data_ptr(), ptr(sums), ptr(scratch), nbytes,
                                      _stream(x.hi.device))
    _lib.check(code, "stp3_dw_fwd")
    return out


def se_proj_weight_elems(cin: int, cout: int) -> int:
    return int(_lib.lib().stp3_se_proj_weight_elems(cin, cout))


def se_chunks(cout: int) -> List[Tuple[int, int, int]]:
    """(first output channel, channels, bn) of the 128-column chunks a projection runs as (stp3_se_gate's layout)."""
    return [(n0, min(128, cout - n0), 128 if cout - n0 > 64 else 64) for n0 in range(0, cout, 128)]


def se_gate(sums: torch.Tensor, hw: int, C: int, w_r, b_r, w_e, b_e, w_proj: torch.Tensor,
            gate: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Squeeze-excite gate of every image folded into per-image projection weights: returns (n_img,
    se_proj_weight_elems(C, cout)) bf16 -- W_proj . diag(gate_img), packed hi/lo in se_chunks(cout) column chunks.
    gate: optional (n_img, C) fp32 destination of the gate itself (allocated when not given)."""
    n_img = sums.shape[0]
    R, cout = w_r.shape[0], w_proj.shape[0]
    assert w_r.shape == (R, C) and w_e.shape == (C, R) and w_proj.shape == (cout, C) and sums.shape[1] >= C
    for t in (sums, w_r, b_r, w_e, b_e, w_proj) + ((gate,) if gate is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    if gate is None:
        gate = torch.empty((n_img, C), dtype=torch.float32, device=sums.device)
    assert gate.shape == (n_img, C)
    w_img = torch.empty((n_img, se_proj_weight_elems(C, cout)), dtype=torch.bfloat16, device=sums.device)
    with torch.cuda.device(sums.device):
        code = _lib.lib().stp3_se_gate(sums.data_ptr(), sums.shape[1], n_img, C, 1.0 / hw, w_r.data_ptr(),
                                       b_r.data_ptr(), R, w_e.data_ptr(), b_e.data_ptr(), w_proj.data_ptr(), cout,
                                       gate.data_ptr(), w_img.data_ptr(),
                                       _stream(sums.device))
    _lib.check(code, "stp3_se_gate")
    return w_img


# ------------------------------------------------------------------------------------------------ prediction stage
# A slot is (HL, first channel, first frame): the channels [coff, coff + C) of frames [t0, t0 + T) of every sample of
# an HL buffer, where the call processes T frames of each of the buffer's B samples (stp3_hl_slot).
def _slot(v, C: int, T: int, bhw: Tuple[int, int, int]) -> "_lib.HlSlot":
    """The stp3_hl_slot of v for a call over B samples of T frames of H x W pixels (bhw = (B, H, W)): the kernels index
    every slot of a call with those dimensions, so each buffer must have them."""
    x, coff, t0 = (v + (0, 0))[:3] if isinstance(v, tuple) else (v, 0, 0)
    assert x.lo is not None and x.hi.is_contiguous() and x.lo.is_contiguous() and x.hi.dtype == torch.bfloat16
    assert x.lo.shape == x.hi.shape and x.lo.dtype == torch.bfloat16
    assert (x.hi.shape[0],) + tuple(x.hi.shape[2:4]) == tuple(bhw), (x.hi.shape, bhw)
    assert coff + C <= x.hi.shape[-1] and t0 + T <= x.hi.shape[1], (coff, C, x.hi.shape, t0, T)
    return _lib.HlSlot(x.hi.data_ptr(), x.lo.data_ptr(), x.hi.shape[-1], coff, x.hi.shape[1], t0)


def _dims(v, T: Optional[int]):
    x, t0 = (v[0], (v + (0, 0))[2]) if isinstance(v, tuple) else (v, 0)
    B, Tt, H, W, _ = x.hi.shape
    return B, (T if T is not None else Tt - t0), H, W, x.hi.device


def gru_gates(r, h, out, C: int, T: Optional[int] = None):
    """out = (1 - sigmoid(r)) * h over C channels (stp3_gru_gates); r, h, out are HLs or slots (HL, coff[, t0])."""
    B, T, H, W, dev = _dims(r, T)
    bhw = (B, H, W)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_gru_gates(_slot(r, C, T, bhw), _slot(h, C, T, bhw), _slot(out, C, T, bhw), B, T, H * W,
                                         C, _stream(dev))
    _lib.check(code, "stp3_gru_gates")


def gru_update(u, h, h_tilde, out, C: int, out2=None, T: Optional[int] = None):
    """out [, out2] = (1 - s) * h + s * h_tilde, s = sigmoid(u) (stp3_gru_update)."""
    B, T, H, W, dev = _dims(u, T)
    bhw = (B, H, W)
    o2 = ctypes.byref(_slot(out2, C, T, bhw)) if out2 is not None else None
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_gru_update(_slot(u, C, T, bhw), _slot(h, C, T, bhw), _slot(h_tilde, C, T, bhw),
                                          _slot(out, C, T, bhw), o2, B, T, H * W, C, _stream(dev))
    _lib.check(code, "stp3_gru_update")


def channel_norm_act(x, out, C: int, ln: Optional[Tuple[torch.Tensor, torch.Tensor, float]] = None, gelu: bool = False,
                     y=None, gelu_y: bool = False, T: Optional[int] = None):
    """out = [gelu]([LN](x)) + [gelu](y) per pixel over C channels; ln = (gamma, beta, eps) (stp3_channel_norm_act)."""
    B, T, H, W, dev = _dims(x, T)
    bhw = (B, H, W)
    g, b, eps = ln if ln is not None else (None, None, 0.0)
    ys = ctypes.byref(_slot(y, C, T, bhw)) if y is not None else None
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_channel_norm_act(_slot(x, C, T, bhw), g.data_ptr() if g is not None else None,
                                                b.data_ptr() if b is not None else None, eps, int(gelu), ys,
                                                int(gelu_y), _slot(out, C, T, bhw), B, T, H * W, C, _stream(dev))
    _lib.check(code, "stp3_channel_norm_act")


def dw_ln(x, w: torch.Tensor, b: torch.Tensor, k: int, ln: Tuple[torch.Tensor, torch.Tensor, float], out, C: int,
          T: Optional[int] = None):
    """out = LN(depthwise k x k (x) + b), w (k*k, C) fp32 (stp3_dw_ln)."""
    B, T, H, W, dev = _dims(x, T)
    bhw = (B, H, W)
    g, beta, eps = ln
    for t in (w, b, g, beta):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert w.shape == (k * k, C) and b.numel() == C
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_dw_ln(_slot(x, C, T, bhw), w.data_ptr(), b.data_ptr(), k, g.data_ptr(), beta.data_ptr(),
                                     eps, _slot(out, C, T, bhw), B, T, H, W, C, _stream(dev))
    _lib.check(code, "stp3_dw_ln")


def trust_mix(t, w: torch.Tensor, s1, s2, dsts, C: int, T: Optional[int] = None):
    """p = softmax(w t), every slot of dsts = s2 * p0 + s1 * p1 (stp3_trust_mix); w (2, C) fp32."""
    B, T, H, W, dev = _dims(t, T)
    bhw = (B, H, W)
    assert w.shape == (2, C) and w.dtype == torch.float32 and w.is_contiguous()
    arr = (_lib.HlSlot * len(dsts))(*[_slot(d, C, T, bhw) for d in dsts])
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_trust_mix(_slot(t, C, T, bhw), w.data_ptr(), _slot(s1, C, T, bhw), _slot(s2, C, T, bhw),
                                         arr, len(dsts), B, T, H * W, C, _stream(dev))
    _lib.check(code, "stp3_trust_mix")


def maxpool2_pad(x: HL, out: Optional[HL] = None) -> HL:
    """2x2 max pool of every channel after zero-padding an odd H / W by one (stp3_maxpool2_pad)."""
    B, T, H, W, cs = x.hi.shape
    if out is None:
        out = HL.empty(B, T, (H + 1) // 2, (W + 1) // 2, x.c, x.hi.device, cp=cs)
    assert out.hi.shape[:4] == (B, T, (H + 1) // 2, (W + 1) // 2)
    o = _slot(out, cs, T, (B, (H + 1) // 2, (W + 1) // 2))
    with torch.cuda.device(x.hi.device):
        code = _lib.lib().stp3_maxpool2_pad(_slot(x, cs, T, (B, H, W)), o, B, T, H, W, cs, _stream(x.hi.device))
    _lib.check(code, "stp3_maxpool2_pad")
    return out


def hl_copy(src, dst, C: int, T: Optional[int] = None):
    """dst = src over C channels (stp3_hl_copy)."""
    B, T, H, W, dev = _dims(src, T)
    bhw = (B, H, W)
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_hl_copy(_slot(src, C, T, bhw), _slot(dst, C, T, bhw), B, T, H * W, C, _stream(dev))
    _lib.check(code, "stp3_hl_copy")


def hl_broadcast(vec: torch.Tensor, dst, C: int, T: Optional[int] = None):
    """dst[img, pixel, :C] = vec[img, :C] with vec (B*T, >= C) fp32 (stp3_hl_broadcast)."""
    B, T, H, W, dev = _dims(dst, T)
    bhw = (B, H, W)
    assert vec.dtype == torch.float32 and vec.is_contiguous() and vec.shape[0] == B * T and vec.shape[1] >= C
    with torch.cuda.device(dev):
        code = _lib.lib().stp3_hl_broadcast(vec.data_ptr(), vec.shape[1], _slot(dst, C, T, bhw), B, T, H * W, C, _stream(dev))
    _lib.check(code, "stp3_hl_broadcast")
