"""GPU, two processes: the train-mode Decoder, DeepLabHead, TemporalModel and UpsamplingConcat after
nn.SyncBatchNorm.convert_sync_batchnorm, with a global batch split 2 + 1 and 2 + 2 over two ranks, against the same module
with plain BatchNorm on the whole batch in this process.  The ranks run in spawned children that are always joined (no
process group ever exists in the pytest process, whose refusal tests expect none): NCCL with one GPU per rank when
there are two, else gloo with both ranks on cuda:0 (its CUDA all-gather carries the BatchNorm records).  Each rank's
loss is its own sum scaled by the world size, so the DDP-averaged gradients are those of the global batch's loss."""
import copy
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import torch_dense as TD
from stp3_b200.layers import convolutions as CV

pytestmark = pytest.mark.gpu
WORLD = 2


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rel_max(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _no_dropout(m):
    # dropout masks depend on where an element sits in its launch, so a split batch draws other masks
    for d in m.modules():
        if isinstance(d, torch.nn.Dropout):
            d.p = 0.0
    return m


def build(kind):
    """-> (module on CPU in train mode, global inputs (batch first), loss weights, forward(module, inputs) -> tensors)"""
    if kind == "decoder":
        from tests.test_decoder_train_gpu import GATES_PERCEIVE, make_decoder
        m = make_decoder(GATES_PERCEIVE)
        fwd = lambda mod, x: [v for v in mod(x[0]).values() if v is not None]        # noqa: E731
        inputs = [gauss((4, 3, 64, 48, 64), 6)]
    elif kind == "deeplab":
        from tests.test_deeplab_train_gpu import make_head
        m = make_head(64, 64, 128)
        fwd = lambda mod, x: [mod(x[0])]                                             # noqa: E731
        inputs = [gauss((4, 64, 48, 64), 5)]
    elif kind == "temporal":
        from tests.test_temporal_train_gpu import make_model
        m = make_model(70, 6, 3, 48, 64)
        fwd = lambda mod, x: [mod(x[0], x[1].flatten(0, 1))]                        # noqa: E731
        inputs = [gauss((4, 3, 64, 48, 64), 5), gauss((4, 3, 6), 6)]
    else:
        m = TD.init_exact(CV.UpsamplingConcat(96, 64), seed=4).train()
        fwd = lambda mod, x: [mod(x[0], x[1])]                                       # noqa: E731
        inputs = [gauss((4, 64, 12, 16), 5), gauss((4, 32, 24, 32), 6)]
    return _no_dropout(m), inputs, fwd


def _worker(rank, port, kind, counts, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    nccl = torch.cuda.device_count() >= WORLD
    dev = torch.device(f"cuda:{rank if nccl else 0}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=WORLD)
    try:
        m, inputs, fwd = build(kind)
        a = sum(counts[:rank])
        local = [t[a:a + counts[rank]] for t in inputs]
        mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).to(dev)
        # the loss weights of the whole batch, restricted to this rank's images
        outs = fwd(mod, [t.to(dev) for t in local])
        loss = 0
        for i, o in enumerate(outs):
            G = gauss((sum(counts), *o.shape[1:]), 40 + i).to(dev)
            loss = loss + (o * G[a:a + o.shape[0]]).sum() * WORLD
        loss.backward()
        grads = {}
        for k, p in mod.named_parameters():
            g = p.grad.clone()
            dist.all_reduce(g)                         # what DDP does with every gradient
            grads[k] = (g / WORLD).cpu().numpy()
        bufs = {k: b.cpu().numpy() for k, b in mod.named_buffers()}
        # numpy arrays travel by value: a torch tensor would be fetched from this process after it has exited
        q.put((rank, [o.detach().cpu().numpy() for o in outs], grads, bufs))
    finally:
        dist.destroy_process_group()


def run_ranks(kind, counts, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, port, kind, counts, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=600) for _ in procs), key=lambda t: t[0])
        res = [(r, [torch.from_numpy(o) for o in outs], {k: torch.from_numpy(v) for k, v in grads.items()},
                {k: torch.from_numpy(v) for k, v in bufs.items()}) for r, outs, grads, bufs in res]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return res


@pytest.mark.parametrize("counts", [(2, 1), (2, 2)])
@pytest.mark.parametrize("kind", ["decoder", "deeplab", "temporal", "upsampling_concat"])
def test_two_ranks_match_one_process_on_the_global_batch(kind, counts):
    port = 29700 + 10 * ["decoder", "deeplab", "temporal", "upsampling_concat"].index(kind) + counts[1]
    res = run_ranks(kind, list(counts), port)
    # one process, plain BatchNorm, the whole batch
    m, inputs, fwd = build(kind)
    mod = copy.deepcopy(m).cuda()
    outs = fwd(mod, [t[:sum(counts)].cuda() for t in inputs])
    loss = sum((o * gauss(tuple(o.shape), 40 + i).cuda()).sum() for i, o in enumerate(outs))
    loss.backward()
    torch.cuda.synchronize()
    worst = {}
    for i, o in enumerate(outs):
        got = torch.cat([r[1][i] for r in res])
        worst[f"out{i}"] = rel_max(got, o.detach())
    for k, b in mod.named_buffers():
        b0, b1 = res[0][3][k], res[1][3][k]
        assert torch.equal(b0, b1), k                         # every rank holds the same running statistics
        if k.endswith("num_batches_tracked"):
            assert int(b0) == int(b), k
        else:
            worst[k] = rel_max(b0, b)
    from tests.test_decoder_train_gpu import ZERO_GRAD
    gmax = max(p.grad.abs().max().item() for p in mod.parameters())
    for k, p in mod.named_parameters():
        assert torch.equal(res[0][2][k], res[1][2][k]), k
        if kind == "decoder" and k in ZERO_GRAD:
            # exactly zero (a train-mode BatchNorm follows): checked against the model's largest gradient, as there
            assert res[0][2][k].abs().max().item() < 1e-5 * gmax, k
            continue
        worst[f"grad.{k}"] = rel_max(res[0][2][k], p.grad)
    print(kind, counts, max(worst.items(), key=lambda kv: kv[1]))
    assert max(v for k, v in worst.items() if k.startswith("out")) <= 1e-5, worst
    assert max(v for k, v in worst.items() if k.startswith("running") or ".running" in k) <= 1e-6, worst
    assert max(v for k, v in worst.items() if k.startswith("grad.")) <= 2.5e-4, worst
