"""GPU, one process: the SyncBatchNorm entry points (stp3_bn_local_moments / stp3_bn_merge_finalize and the backward's
stp3_bn_bwd_local_sums / stp3_bn_bwd_merge_sums / stp3_bn_bwd_apply_global) on W in {1, 2, 3, 4} uneven row slices of
one tensor, each slice's record written into its row of one buffer (what the all-gather leaves on every rank), against
the fp64 statistics and the fp64 SyncBatchNorm backward of the whole tensor."""
import pytest
import torch

from stp3_b200 import _lib, dense_train as T
from oracle import torch_dense as TD

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_ROWS = 6 * 48 * 64


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rel_max(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def elem_rel(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return (got - ref).abs() / ref.abs()


def split(n, W):
    """W uneven, non-empty slices of n rows: [(start, count)]."""
    w = torch.arange(1, W + 1, dtype=torch.float64)
    counts = (w / w.sum() * n).floor().long()
    counts[-1] += n - int(counts.sum())
    starts = torch.cumsum(counts, 0) - counts
    return list(zip(starts.tolist(), counts.tolist()))


def data(C, seed):
    """(N_ROWS, C) fp32 with a channel whose |mean| is 1e3 x its std (the last one)."""
    x = gauss((N_ROWS, C), seed) * 2.0 + 0.5
    x[:, -1] = x[:, -1] * 0.01 + 10.0
    return x.to(DEV).contiguous()


def _s():
    return torch.cuda.current_stream().cuda_stream


def sync_stats(x, slices, eps=1e-5, momentum=0.1, rm=None, rv=None):
    L = _lib.lib()
    C = x.shape[1]
    rec = torch.full((len(slices), 4, C), float("nan"), dtype=torch.float64, device=DEV)
    for r, (a, n) in enumerate(slices):
        nbytes = L.stp3_bn_scratch_bytes(n, C)
        scratch = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
        assert L.stp3_bn_local_moments(x[a:a + n].data_ptr(), n, C, C, rec[r].data_ptr(), scratch.data_ptr(), nbytes,
                                       _s()) == 0
    mean, var, invstd = (torch.empty(C, device=DEV) for _ in range(3))
    assert L.stp3_bn_merge_finalize(rec.data_ptr(), len(slices), C, eps, momentum, T._p(rm), T._p(rv),
                                    mean.data_ptr(), var.data_ptr(), invstd.data_ptr(), _s()) == 0
    return rec, mean, var, invstd


def sync_backward(g, y, x, slices, mean, invstd, gamma):
    """-> (dx, per-slice local (sum_g, sum_gx) fp32, merged (sum_g, sum_gx))"""
    L = _lib.lib()
    C = x.shape[1]
    rec = torch.full((len(slices), 2, C), float("nan"), dtype=torch.float64, device=DEV)
    local = []
    for r, (a, n) in enumerate(slices):
        nbytes = L.stp3_bn_scratch_bytes(n, C)
        scratch = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
        assert L.stp3_bn_bwd_local_sums(g[a:a + n].data_ptr(), C, y[a:a + n].data_ptr(), C, x[a:a + n].data_ptr(), C,
                                        mean.data_ptr(), invstd.data_ptr(), n, C, rec[r].data_ptr(), scratch.data_ptr(),
                                        nbytes, _s()) == 0
        sg, sgx = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
        assert L.stp3_bn_bwd_merge_sums(rec[r].data_ptr(), 1, C, sg.data_ptr(), sgx.data_ptr(), _s()) == 0
        local.append((sg, sgx))
    tg, tgx = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    assert L.stp3_bn_bwd_merge_sums(rec.data_ptr(), len(slices), C, tg.data_ptr(), tgx.data_ptr(), _s()) == 0
    dx = torch.full_like(x, float("nan"))
    for a, n in slices:
        assert L.stp3_bn_bwd_apply_global(g[a:a + n].data_ptr(), C, y[a:a + n].data_ptr(), C, x[a:a + n].data_ptr(), C,
                                          mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), tg.data_ptr(),
                                          tgx.data_ptr(), n, x.shape[0], C, dx[a:a + n].data_ptr(), C, None, 0,
                                          _s()) == 0
    return dx, local, (tg, tgx)


CHANNELS = [21, 23, 35, 44, 67]


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("C", CHANNELS)
def test_merged_statistics_match_fp64(C, W):
    x = data(C, 3)
    slices = split(N_ROWS, W)
    rm, rv = (gauss((C,), 4) * 0.1).to(DEV), (gauss((C,), 5).abs() + 0.5).to(DEV)
    rm0, rv0 = rm.clone(), rv.clone()
    rec, mean, var, invstd = sync_stats(x, slices, 1e-5, 0.1, rm, rv)
    torch.cuda.synchronize()
    xd = x.double().cpu()
    mu, vb = xd.mean(0), xd.var(0, unbiased=False)
    # the bar of DESIGN.md 3.7 (one fp32 rounding), channel by channel: the large-mean channel keeps it too
    assert float(elem_rel(mean, mu).max()) <= 7e-8
    assert float(elem_rel(var, vb).max()) <= 7e-8
    assert float(elem_rel(invstd, 1 / (vb + 1e-5).sqrt()).max()) <= 7e-8
    assert rel_max(rm, 0.9 * rm0.double().cpu() + 0.1 * mu) <= 1e-6
    assert rel_max(rv, 0.9 * rv0.double().cpu() + 0.1 * xd.var(0, unbiased=True)) <= 1e-6
    # the counts are part of the record
    assert rec[:, 0, 0].tolist() == [float(n) for _, n in slices]
    # two launches: the same bits
    rm2, rv2 = rm0.clone(), rv0.clone()
    _, m2, v2, i2 = sync_stats(x, slices, 1e-5, 0.1, rm2, rv2)
    assert torch.equal(m2, mean) and torch.equal(v2, var) and torch.equal(i2, invstd)
    assert torch.equal(rm2, rm) and torch.equal(rv2, rv)
    if W == 1:
        rm3, rv3 = rm0.clone(), rv0.clone()
        st = T.bn_stats(x.view(1, 1, N_ROWS, C), 1e-5, 0.1, rm3, rv3)
        assert torch.equal(st.mean, mean) and torch.equal(st.var, var) and torch.equal(st.invstd, invstd)
        assert torch.equal(rm3, rm) and torch.equal(rv3, rv)


@pytest.mark.parametrize("C", CHANNELS)
def test_merge_is_order_independent_up_to_fp64_rounding(C):
    """Permuting the rows across the slices moves the statistics by fp64 rounding only."""
    x = data(C, 7)
    slices = split(N_ROWS, 3)
    _, mean, var, _ = sync_stats(x, slices)
    perm = torch.randperm(N_ROWS, generator=torch.Generator().manual_seed(1)).to(DEV)
    _, mean_p, var_p, _ = sync_stats(x[perm].contiguous(), slices)
    # fp64 sums in another order: at most one fp32 rounding flips
    assert float(elem_rel(mean_p, mean).max()) <= 1.2e-7
    assert float(elem_rel(var_p, var).max()) <= 1.2e-7


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("C", CHANNELS)
def test_backward_matches_fp64_syncbn(C, W):
    x = data(C, 11)
    slices = split(N_ROWS, W)
    _, mean, var, invstd = sync_stats(x, slices)
    gamma, beta = (gauss((C,), 12) * 0.3 + 1.0).to(DEV), (gauss((C,), 13) * 0.1).to(DEV)
    st = T.BNStats(mean, var, invstd, N_ROWS)
    y, _ = T.bn_apply(x.view(1, 1, N_ROWS, C), st, gamma, beta, relu=True, hl=False)
    y = y.view(N_ROWS, C)
    g = gauss((N_ROWS, C), 14).to(DEV)
    dx, local, (tg, tgx) = sync_backward(g, y, x, slices, mean, invstd, gamma)
    torch.cuda.synchronize()
    # fp64 SyncBatchNorm backward on the whole tensor, with the ReLU mask of the kernels' own forward
    xd = x.double().cpu().requires_grad_(True)
    bn = torch.nn.BatchNorm1d(C, momentum=0.1).double()
    with torch.no_grad():
        bn.weight.copy_(gamma.cpu()); bn.bias.copy_(beta.cpu())
    z = bn(xd)
    gd = torch.where(y.cpu() > 0, g.cpu(), torch.zeros_like(g.cpu())).double()
    gx, = torch.autograd.grad(z, xd, gd)
    assert rel_max(dx, gx) < 1e-4                                       # the dgrad bar of bn_backward's test
    # per-slice sums: dbeta / dgamma of that rank; their merge is the whole tensor's.  x-hat is formed in fp32 from the
    # fp32 mean and invstd (~1e-7 of each term), and a slice's sum cancels more than the whole tensor's: 5e-5 of max
    xhat = (xd.detach() - xd.detach().mean(0)) / (xd.detach().var(0, unbiased=False) + 1e-5).sqrt()
    for (a, n), (sg, sgx) in zip(slices, local):
        assert rel_max(sg, gd[a:a + n].sum(0)) < 5e-5
        assert rel_max(sgx, (gd[a:a + n] * xhat[a:a + n]).sum(0)) < 5e-5
    assert rel_max(tg, gd.sum(0)) < 1e-5 and rel_max(tgx, (gd * xhat).sum(0)) < 1e-5
    dx2, local2, (tg2, tgx2) = sync_backward(g, y, x, slices, mean, invstd, gamma)
    assert torch.equal(dx2, dx) and torch.equal(tg2, tg) and torch.equal(tgx2, tgx)
    if W == 1:
        st1 = T.BNStats(mean, var, invstd, N_ROWS)
        dx1, sgx1, sg1, _ = T.bn_backward(g.view(1, 1, N_ROWS, C), x.view(1, 1, N_ROWS, C), st1, gamma,
                                          y.view(1, 1, N_ROWS, C))
        assert torch.equal(sg1, local[0][0]) and torch.equal(sgx1, local[0][1])
        assert torch.equal(sg1, tg) and torch.equal(sgx1, tgx)
        assert torch.equal(dx1.view(N_ROWS, C), dx)


def test_argument_errors():
    L = _lib.lib()
    fake = 1 << 20
    assert L.stp3_bn_local_moments(fake, 0, 8, 8, fake, fake, 1 << 20, None) == -1
    assert L.stp3_bn_merge_finalize(fake, 0, 8, 1e-5, 0.1, None, None, fake, fake, fake, None) == -1
    assert L.stp3_bn_merge_finalize(fake, 2, 8, 1e-5, 0.1, fake, None, fake, fake, fake, None) == -1
    assert L.stp3_bn_bwd_apply_global(fake, 8, None, 0, fake, 8, fake, fake, fake, fake, fake, 10, 9, 8, fake, 8,
                                      None, 0, None) == -1
    assert b"n_total" in L.stp3_last_error()
