"""Train-step time of the decoder + temporal model under DDP on two GPUs (one NCCL rank each), with SyncBatchNorm
(convert_sync_batchnorm: ~2 small all-gathers per BatchNorm and step) and with plain BatchNorm (local statistics), on
the same per-rank batch (B=1, S=3, 64 x 200 x 200).  Median over timed steps of CUDA events around forward + backward
+ DDP's gradient all-reduce, max over ranks; the two variants alternate within one run.  Prints one JSON line with the
GPU name and power limit read in the same run.  Needs two GPUs: with fewer it exits with an error.

    python tools/syncbn_train_bench.py [--steps 20] [--warmup 3] [--hw 200 200]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import torch_dense as TD  # noqa: E402
from stp3_b200.models.decoder import Decoder  # noqa: E402
from stp3_b200.models.temporal_model import TemporalModel  # noqa: E402

GATES = dict(perceive_hdmap=True, predict_pedestrian=True, predict_instance=False, predict_future_flow=False,
             planning=False)
WORLD = 2


class Net(torch.nn.Module):
    def __init__(self, hw):
        super().__init__()
        self.tm = TemporalModel(64, 3, hw, start_out_channels=64)
        self.dec = Decoder(64, 2, 3, 2, GATES)

    def forward(self, x):
        y = self.tm(x)
        return [v for v in self.dec(y).values() if v is not None]


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:                               # noqa: BLE001  (reported as unknown)
        power = None
    return name, power


def _worker(rank, args, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = "29850"
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=WORLD)
    try:
        H, W = args.hw
        x = TD.exact_gauss((1, 3, 64, H, W), torch.Generator().manual_seed(5 + rank)).to(dev)
        models = {}
        for sync in (False, True):
            net = TD.init_exact(Net((H, W)), seed=3).train()
            if sync:
                net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(net)
            models[sync] = torch.nn.parallel.DistributedDataParallel(net.to(dev), device_ids=[rank])
        times = {False: [], True: []}

        def step(m):
            sum(o.float().square().mean() for o in m(x)).backward()
        for sync, m in models.items():
            for _ in range(args.warmup):
                step(m)
        for i in range(args.steps):
            for sync in ((False, True) if i % 2 == 0 else (True, False)):
                dist.barrier()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step(models[sync])
                b.record()
                b.synchronize()
                times[sync].append(a.elapsed_time(b))
        med = torch.tensor([statistics.median(times[False]), statistics.median(times[True])], device=dev)
        dist.all_reduce(med, op=dist.ReduceOp.MAX)
        if rank == 0:
            q.put(med.tolist())
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--hw", type=int, nargs=2, default=(200, 200))
    args = ap.parse_args()
    if torch.cuda.device_count() < WORLD:
        sys.exit(f"syncbn_train_bench: needs {WORLD} GPUs, found {torch.cuda.device_count()}")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, args, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    plain, sync = q.get(timeout=1800)
    for p in procs:
        p.join()
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit_w": power, "world": WORLD, "per_rank_batch": 1, "S": 3,
                      "hw": list(args.hw), "steps": args.steps, "step_ms_plain_bn": round(plain, 3),
                      "step_ms_sync_bn": round(sync, 3), "sync_overhead": round(sync / plain - 1.0, 4)}))


if __name__ == "__main__":
    main()
