"""Multi-GPU plumbing of the hot path: one process per GPU (torchrun), batch axis sharded, no data-path collective.

Every sample is independent through lift-splat -> temporal model -> decoder (the reference loops over the batch,
stp3.py:265, and eval-mode BatchNorm has no cross-sample coupling), so ranks simply own disjoint slices of the global
batch.  torch.distributed (NCCL on the GPUs, gloo in the CPU tests) is used for rendezvous, the barrier around timed
regions, the max-over-ranks reduction of device times and, when a single consumer wants them, gathering the logits.
Training under SyncBatchNorm adds one small all-gather per BatchNorm and direction (all_gather_rows).
"""
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist


def world() -> Tuple[int, int]:
    """(rank, world_size); (0, 1) when torch.distributed is not initialised."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_batch(global_batch: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous slice [start, start+count) of the global batch owned by `rank` (sizes differ by at most one)."""
    if not 0 <= rank < world_size:
        raise ValueError("rank out of range")
    base, extra = divmod(global_batch, world_size)
    start = rank * base + min(rank, extra)
    return start, base + (1 if rank < extra else 0)


def barrier():
    if dist.is_available() and dist.is_initialized():
        dist.barrier()


def max_over_ranks(value: float, device: Optional[torch.device] = None) -> float:
    """Slowest rank decides: every multi-GPU time reported by bench.py is the max over ranks."""
    rank, ws = world()
    if ws == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_outputs(outputs: Dict[str, Optional[torch.Tensor]], global_batch: int) -> Dict[str, Optional[torch.Tensor]]:
    """All-gather the per-rank logits (dim 0 = this rank's samples) into global-batch order on every rank.
    Only needed when ONE consumer wants the whole batch; the forward path itself needs no collective."""
    rank, ws = world()
    if ws == 1:
        return outputs
    counts = [shard_batch(global_batch, r, ws)[1] for r in range(ws)]
    out = {}
    for key, t in outputs.items():
        if t is None:
            out[key] = None
            continue
        pad = max(counts) - t.shape[0]
        tp = torch.cat([t, t.new_zeros((pad, *t.shape[1:]))]) if pad else t
        parts = [torch.empty_like(tp) for _ in range(ws)]
        dist.all_gather(parts, tp.contiguous())
        out[key] = torch.cat([p[:c] for p, c in zip(parts, counts)])
    return out


def all_gather_frames(local: torch.Tensor, n_frames: int) -> torch.Tensor:
    """The ONE collective of the frame-sharded mode: local (f_count, X, Y, C) raw BEV frames of this rank ->
    (n_frames, X, Y, C) on every rank, in flat-frame order (rank r owns shard_batch(n_frames, r, world))."""
    rank, ws = world()
    if ws == 1:
        return local
    counts = [shard_batch(n_frames, r, ws)[1] for r in range(ws)]
    cmax = max(counts)
    pad = cmax - local.shape[0]
    lp = torch.cat([local, local.new_zeros((pad, *local.shape[1:]))]) if pad else local.contiguous()
    gathered = torch.empty((ws * cmax, *local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(gathered, lp)
    if all(c == cmax for c in counts):
        return gathered
    return torch.cat([gathered[r * cmax:r * cmax + c] for r, c in enumerate(counts)])


def all_gather_rows(buf: torch.Tensor, group=None) -> torch.Tensor:
    """buf (world, ...) with this rank's row written -> every rank's row, in rank order, in place (the list form of
    all_gather: NCCL, and gloo's CUDA allgather).  The SyncBatchNorm records' exchange (dense_train.bn_stats_module)."""
    rows = list(buf.unbind(0))
    dist.all_gather(rows, rows[dist.get_rank(group)], group=group)
    return buf


class PeerFrameBuffer:
    """Every rank's (n_frames, X, Y, C) fp32 gather buffer in symmetric memory (torch.distributed._symmetric_memory: CUDA
    peer mappings over NVLink), so that the frame-sharded lift-splat can store its frames into all ranks' buffers from
    its own epilogue (stp3_lift_splat_fwd with n_peers > 0) instead of running a separate all-gather.
    barrier() = device-side cross-rank barrier on the current stream (signal pads of the symmetric allocation)."""

    def __init__(self, n_frames: int, X: int, Y: int, C: int, device, group=None):
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        self.buf = symm.empty((n_frames, X, Y, C), dtype=torch.float32, device=device)
        self.hdl = symm.rendezvous(self.buf, group)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]

    def barrier(self):
        self.hdl.barrier()
