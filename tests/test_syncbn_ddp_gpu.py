"""GPU, two ranks on two GPUs (NCCL; skipped with fewer): the reference's recipe end to end -- a small STP3 with an
injected torch trunk, convert_sync_batchnorm, DistributedDataParallel(find_unused_parameters=False), two SGD steps on a
global batch of 2 split 1 + 1, then model.eval().  Parameters stay bitwise equal across ranks and the eval logits match
the single-process plain-BatchNorm model trained on the global batch.  A native-trunk model (frozen trunk,
train_heads()) completes two steps too.  Ranks run in spawned children that are always joined."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_encoder_train_gpu import ConvTrunk, LCFG, gauss, loss_of, small_stp3

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (one NCCL rank each)")]
WORLD = 2


def images(n):
    return gauss((n, 3, 2, 3, *LCFG.final_dim), 3)


def train_two_steps(model, image, inp, dev, scale):
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-2)
    snaps = []
    for _ in range(2):
        opt.zero_grad()
        out = model(image.to(dev), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        (loss_of(out) * scale).backward()
        opt.step()
        snaps.append({k: p.detach().cpu().numpy().copy() for k, p in model.named_parameters()})
    return snaps


def eval_logits(model, image, inp, dev):
    model.eval()
    with torch.no_grad():
        out = model(image.to(dev), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    return {k: out[k].float().cpu().numpy() for k in ("segmentation", "pedestrian", "hdmap")}


def _worker(rank, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=WORLD)
    try:
        model, inp = small_stp3(ConvTrunk())
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model).to(dev).train()
        for d in model.modules():
            if isinstance(d, torch.nn.Dropout):
                d.p = 0.0
        ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[rank], find_unused_parameters=False)
        img = images(WORLD)[rank:rank + 1]
        # loss_of takes means over the local batch of one: DDP's average over ranks is the global batch's loss
        snaps = train_two_steps(ddp, img, inp, dev, 1.0)
        logits = eval_logits(model, images(WORLD), inp, dev)
        # the frozen native trunk recipe under DDP
        nat, _ = small_stp3("native")
        nat = torch.nn.SyncBatchNorm.convert_sync_batchnorm(nat).to(dev)
        nat.eval()
        nat.encoder.backbone.requires_grad_(False)
        nat.encoder.train_heads()
        nat.temporal_model.train()
        nat.decoder.train()
        ddp_nat = torch.nn.parallel.DistributedDataParallel(nat, device_ids=[rank], find_unused_parameters=False)
        train_two_steps(ddp_nat, img, inp, dev, 1.0)
        q.put((rank, snaps, logits))
    finally:
        dist.destroy_process_group()


def test_ddp_sync_batchnorm_two_steps_match_one_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 29800, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=900) for _ in procs), key=lambda t: t[0])
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    for s0, s1 in zip(res[0][1], res[1][1]):
        for k in s0:
            assert (s0[k] == s1[k]).all(), k
    # one process, plain BatchNorm, the global batch
    model, inp = small_stp3(ConvTrunk())
    for d in model.modules():
        if isinstance(d, torch.nn.Dropout):
            d.p = 0.0
    model.train()
    dev = torch.device("cuda:0")
    train_two_steps(model, images(WORLD), inp, dev, 1.0)
    ref = eval_logits(model, images(WORLD), inp, dev)
    for k, v in ref.items():
        e = float(abs(res[0][2][k] - v).max() / abs(v).max())
        assert e <= 1e-3, (k, e)
