"""GPU: the memory-bound helpers the dense forward launches around its convolutions (pool_bias, small_linear,
upsample2x_add, the fp32 <-> hi/lo layout conversions, spatial_sum) against plain float64 torch, at parameter values the
modules do not pass today: accumulation, strided output rows, windows at 8 mod 16, channel counts that are not
multiples of the kernels' 32-channel tiles, ragged pixel chunks.  Outside the written windows nothing may change."""
import pytest
import torch
import torch.nn.functional as F

from stp3_b200 import dense

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -1.5e30


def rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(*shape, generator=g) * 2 - 1) * scale).to(DEV)


def rel(got, ref, scale=None):
    ref = ref.double()
    return float((got.double() - ref).abs().max()) / (scale if scale is not None else float(ref.abs().max()))


def hl(x_cl):
    hi, lo = dense.split_hilo(x_cl)
    return dense.HL(hi.contiguous(), lo.contiguous(), x_cl.shape[-1])


@pytest.mark.parametrize("temporal,n_const,accumulate,CO,extra,with_bias", [
    (True, 0, False, 64, 0, True),        # CO >= 64: four slices of output rows
    (False, 6, True, 35, 16, False),      # spatially constant trailing channels, sums rows wider than the spatial C
    (True, 6, False, 130, 8, False),
    (False, 0, True, 128, 0, True),
    (True, 3, True, 20, 40, True),
])
def test_pool_bias(temporal, n_const, accumulate, CO, extra, with_bias):
    B, T, C, R, hw = 2, 3, 70, 35, 37 * 29
    n = B * T
    cs = C - n_const
    sums = rnd(n, cs + extra, seed=1, scale=float(hw)).contiguous()
    const = rnd(n, n_const, seed=2).contiguous() if n_const else None
    W1, b1 = rnd(R, C, seed=3, scale=0.2).contiguous(), rnd(R, seed=4)
    W2 = rnd(CO, R, seed=5, scale=0.2).contiguous()
    bias = rnd(CO + 3, seed=6) if with_bias else None
    co_stride = CO + 5
    out = rnd(n, co_stride, seed=7).contiguous()
    prior = out.clone()
    dense.pool_bias(sums, T, C, hw, temporal, W1, b1, W2, out, accumulate, const=const, bias=bias)
    torch.cuda.synchronize()
    m = sums[:, :cs].double() / hw
    if n_const:
        m = torch.cat([m, const.double()], 1)
    if temporal:
        prev = torch.cat([m[:1], m[:-1]])
        first = (torch.arange(n, device=DEV) % T == 0).view(-1, 1)
        m = torch.where(first, m, (m + prev) / 2)
    v = F.relu(m @ W1.double().t() + b1.double())
    base = prior[:, :CO].double() if accumulate else (bias[:CO].double().expand(n, CO) if with_bias else 0.0)
    ref = base + v @ W2.double().t()
    assert rel(out[:, :CO], ref) < 1e-5
    assert torch.equal(out[:, CO:], prior[:, CO:])


@pytest.mark.parametrize("accumulate,with_bias,co,co_stride", [(False, True, 64, 64), (True, False, 35, 48),
                                                                 (False, False, 130, 136), (True, True, 6, 64)])
def test_small_linear(accumulate, with_bias, co, co_stride):
    n, ci = 6, 6
    x, W = rnd(n, ci, seed=11).contiguous(), rnd(co, ci, seed=12).contiguous()
    bias = rnd(co, seed=13) if with_bias else None
    out = rnd(n, co_stride, seed=14).contiguous()
    prior = out.clone()
    dense.small_linear(x, W, out, accumulate, bias=bias)
    torch.cuda.synchronize()
    base = prior[:, :co].double() if accumulate else (bias.double().expand(n, co) if with_bias else 0.0)
    assert rel(out[:, :co], base + x.double() @ W.double().t()) < 1e-6
    assert torch.equal(out[:, co:], prior[:, co:])


@pytest.mark.parametrize("skip,s_coff,y_coff,c,hw", [(False, 0, 0, 64, (9, 11)), (True, 8, 24, 40, (7, 13)),
                                                     (True, 24, 8, 64, (5, 4)), (False, 0, 40, 16, (1, 6))])
def test_upsample2x_add(skip, s_coff, y_coff, c, hw):
    B, T = 2, 2
    h, w = hw
    x = rnd(B, T, h, w, 72, seed=21)
    s = rnd(B, T, 2 * h, 2 * w, 96, seed=22)
    ys = 112
    out = dense.HL(torch.full((B, T, 2 * h, 2 * w, ys), SENT, dtype=torch.bfloat16, device=DEV),
                   torch.full((B, T, 2 * h, 2 * w, ys), SENT, dtype=torch.bfloat16, device=DEV), ys)
    xh, sh = hl(x), hl(s)
    dense.upsample2x_add(xh, sh if skip else None, c, skip_coff=s_coff, out=out, out_coff=y_coff)
    torch.cuda.synchronize()
    xj = (xh.hi.double() + xh.lo.double())[..., :c].reshape(B * T, h, w, c).permute(0, 3, 1, 2)
    ref = F.interpolate(xj, scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    ref = ref.reshape(B, T, 2 * h, 2 * w, c)
    if skip:
        ref = ref + (sh.hi.double() + sh.lo.double())[..., s_coff:s_coff + c]
    got = out.hi.double() + out.lo.double()
    assert rel(got[..., y_coff:y_coff + c], ref) < 1e-5
    sent = torch.tensor(SENT, dtype=torch.bfloat16, device=DEV)
    for p in (out.hi, out.lo):
        assert bool((p[..., :y_coff] == sent).all()) and bool((p[..., y_coff + c:] == sent).all())


@pytest.mark.parametrize("C,cp,channels_last", [(70, 128, False), (70, 128, True), (13, 64, False), (200, 256, True),
                                                (64, 64, False)])
def test_f32_to_hilo(C, cp, channels_last):
    B, T, H, W = 2, 3, 13, 21
    x = rnd(B, T, H, W, C, seed=31)
    src = x if channels_last else x.permute(0, 1, 4, 2, 3)
    h = dense.from_f32(src.contiguous(), channels_last=channels_last, cp=cp)
    torch.cuda.synchronize()
    assert h.hi.shape == (B, T, H, W, cp)
    hi, lo = dense.split_hilo(x)                      # round to nearest even, like the kernel
    assert torch.equal(h.hi[..., :C], hi) and torch.equal(h.lo[..., :C], lo)
    assert float(h.hi[..., C:].float().abs().max() if cp > C else 0.0) == 0.0
    assert float(h.lo[..., C:].float().abs().max() if cp > C else 0.0) == 0.0


@pytest.mark.parametrize("cs,c_off,C", [(128, 8, 70), (64, 0, 13), (256, 64, 150), (72, 40, 32)])
def test_hilo_to_f32(cs, c_off, C):
    B, T, H, W = 2, 2, 11, 19
    h = hl(rnd(B, T, H, W, cs, seed=41))
    y = dense.to_f32(h, c_off, C)
    torch.cuda.synchronize()
    ref = (h.hi.float() + h.lo.float())[..., c_off:c_off + C].permute(0, 1, 4, 2, 3)
    assert y.shape == (B, T, C, H, W) and torch.equal(y, ref)


@pytest.mark.parametrize("cstride,hw", [(8, (13, 21)), (64, (1, 1)), (200, (37, 29)), (1024, (9, 15)), (120, (16, 8))])
def test_spatial_sum(cstride, hw):
    H, W = hw
    h = hl(rnd(2, 3, H, W, cstride, seed=51, scale=4.0))
    s = dense.spatial_sum(h)
    torch.cuda.synchronize()
    j = h.hi.double() + h.lo.double()
    ref = j.sum(dim=(2, 3)).reshape(6, cstride)
    scale = float(j.abs().sum(dim=(2, 3)).max())
    assert s.shape == (6, cstride) and rel(s, ref, scale) < 1e-6
