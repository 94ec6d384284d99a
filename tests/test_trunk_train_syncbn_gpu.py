"""GPU: the trainable native trunk under SyncBatchNorm -- two ranks over gloo on one GPU (the pattern of
tests/test_syncbn_modules_gpu.py) against one process on the global batch.  The drop-connect draws are pinned: every
call of torch.rand returns this rank's slice of the global batch's values, so both sides drop the same images.
Outputs within 1e-5 of max, running statistics within 1e-6, gradients (summed over the ranks, as DDP sums them up to
its 1 / world) within 2.5e-4 of max, and every rank holds the same running-statistic bits."""
import contextlib
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

WORLD = 2
M, H, W = 4, 48, 64


def build():
    from oracle import efficientnet_oracle as EO
    from stp3_b200.models import efficientnet as EN
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle("b4"), seed=3), "b4")
    nat = EN.EfficientNetTrunk("b4", trainable=True)
    nat.load_state_dict(ora.state_dict(), strict=True)
    for m in nat.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = 0.1
    g = torch.Generator().manual_seed(7)
    x = torch.randn(M, 3, H, W, generator=g)
    g3, g4 = torch.randn(M, 56, 6, 8, generator=g), torch.randn(M, 160, 3, 4, generator=g)
    n_draws = sum(1 for i, b in enumerate(nat._blocks) if b.spec.skip and i > 0)
    U = [torch.rand(M, generator=g) for _ in range(n_draws)]
    return nat.train(), x, g3, g4, U


@contextlib.contextmanager
def pinned_rand(U, a, m):
    """torch.rand(m, ...) inside the trunk returns images [a, a + m) of the global batch's next draw"""
    real, it = torch.rand, iter(U)

    def fake(n, *args, dtype=None, device=None, **kw):
        assert n == m
        return next(it)[a:a + m].to(device=device, dtype=dtype)
    torch.rand = fake
    try:
        yield
    finally:
        torch.rand = real
    assert next(it, None) is None, "the trunk drew fewer masks than it has drop-connect blocks"


def _worker(rank, port, counts, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        nat, x, g3, g4, U = build()
        a, m = sum(counts[:rank]), counts[rank]
        mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(nat).to(dev)
        assert any(isinstance(b, torch.nn.SyncBatchNorm) for b in mod.modules())
        with pinned_rand(U, a, m):
            r3, r4 = mod(x[a:a + m].to(dev))
        ((r3 * g3[a:a + m].to(dev)).sum() + (r4 * g4[a:a + m].to(dev)).sum()).backward()
        grads = {}
        for k, p in mod.named_parameters():
            gsum = p.grad.clone()
            dist.all_reduce(gsum)
            grads[k] = gsum.cpu().numpy()
        bufs = {k: b.cpu().numpy() for k, b in mod.named_buffers()}
        q.put((rank, [r3.detach().cpu().numpy(), r4.detach().cpu().numpy()], grads, bufs))
    finally:
        dist.destroy_process_group()


def run_ranks(counts, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, port, counts, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=600) for _ in procs), key=lambda t: t[0])
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return [(r, [torch.from_numpy(o) for o in outs], {k: torch.from_numpy(v) for k, v in g.items()},
             {k: torch.from_numpy(v) for k, v in b.items()}) for r, outs, g, b in res]


def rel_max(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("counts", [(2, 2), (3, 1)])
def test_two_ranks_match_one_process_on_the_global_batch(counts):
    from tests.test_trunk_train_gpu import zero_grad_params
    res = run_ranks(list(counts), 29800 + counts[1])
    nat, x, g3, g4, U = build()
    mod = nat.cuda()
    with pinned_rand(U, 0, M):
        r3, r4 = mod(x.cuda())
    ((r3 * g3.cuda()).sum() + (r4 * g4.cuda()).sum()).backward()
    torch.cuda.synchronize()
    worst = {}
    for i, o in enumerate((r3, r4)):
        got = torch.cat([r[1][i] for r in res])
        worst[f"reduction_{3 + i}"] = rel_max(got, o.detach())
        assert worst[f"reduction_{3 + i}"] <= 1e-5, worst
    for k, b in mod.named_buffers():
        b0, b1 = res[0][3][k], res[1][3][k]
        assert torch.equal(b0, b1), k
        if k.endswith("num_batches_tracked"):
            assert int(b0) == int(b), k
        else:
            r = rel_max(b0, b)
            worst["running statistics"] = max(worst.get("running statistics", 0.0), r)
            assert r <= 1e-6, (k, r)
    zero = zero_grad_params(mod)
    params = dict(mod.named_parameters())
    for k, p in params.items():
        assert torch.equal(res[0][2][k], res[1][2][k]), k
        got = res[0][2][k].double()
        if k in zero:      # exactly zero in exact arithmetic: held relative to the same layer's weight gradient
            r = float((got - p.grad.double().cpu()).abs().max() / params[zero[k]].grad.abs().max())
        else:
            r = rel_max(got, p.grad)
        worst["gradients"] = max(worst.get("gradients", 0.0), r)
        assert r <= 2.5e-4, (k, r)
    print("worst ratios", counts, worst)
