"""Device time of the two TemporalBlock tails (stp3_block_fused_fwd) at the perceive shape (B=4, T=3, 200 x 200, the
temporal model's 70 -> 64 block with the six ego-motion channels and the projection, then its 64 -> 64 block with the
identity residual), set against what the tile schedule asks of the tensor pipe and of L2.

    python tools/block_bench.py [--reps 100] [--warmup 10] [--schedule p-regs] [--save DIR | --compare DIR]
    python tools/block_bench.py --count-only              # the host-side step / byte counts, no GPU

The counts restate block_fused.cu's schedule on the host from the chain descriptors the blocks pack: one CTA per
tile (--tile, 8x16 by default), a tap group (the three dy taps of a kernel column) skipped when it is padding for the
tile, each executed group moving one activation stage ((tile rows + 2) x tile columns x 64 channels, hi + lo) and each
executed tap one weight stage (the chain's N rows, hi + lo) from L2.  Two schedules are counted:
  p-smem : P in shared memory; all 8 K steps of the aggregation and its two weight blocks per tile; the projection
           loads its own x stage
  p-regs : P in registers; K steps of P that hold no channel are not issued; the aggregation weights stay resident
           (one load per CTA); the projection reads path 2's x stage
--schedule names the schedule of the build being timed.  MACs count the padding of every chain (N and K rounded up)
and the three products of the bf16 hi / lo split.  Prints one JSON line with the GPU name, power limit and the SM clock
sampled during the timed loop.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from head_bench import FLOP_PER_CLK_SM, ClockSampler, gpu_info  # noqa: E402

B, T, H, W = 4, 3, 200, 200
N_CONST = 6                                  # ego-motion channels, spatially constant: per-image biases
SCHEDULES = ("p-smem", "p-regs")


def build_model(dev="cpu"):
    from oracle import torch_dense as TD
    from stp3_b200.models.temporal_model import TemporalModel
    tm = TD.init_exact(TemporalModel(64 + N_CONST, T, (H, W), start_out_channels=64), seed=42).eval().to(dev)
    tm.model[0].n_const = N_CONST
    return tm


def tap_groups(taps):
    """The kernel's tap groups: runs of <= 3 taps with the same (dt, dx) and dy advancing by one."""
    groups, i = [], 0
    while i < len(taps):
        g = 1
        while (g < 3 and i + g < len(taps) and taps[i + g][0] == taps[i][0] and taps[i + g][2] == taps[i][2]
               and taps[i + g][1] == taps[i][1] + g):
            g += 1
        groups.append((taps[i], g))
        i += g
    return groups


def count_block(pb, schedule, th, tw, n_sm):
    """Host restatement of one stp3_block_fused_fwd launch over B*T images of H x W in th x tw tiles."""
    tiles_x, tiles_y = -(-W // tw), -(-H // th)
    m = th * tw
    a_stage = 2 * (th + 2) * tw * 128
    chains = [(c[0], c[2], c[3], (c[6] - c[5]) // 16) for c in pb.chains]     # (src, taps, N, K steps)
    pieces = [v for v in pb.piece_col if v >= 0]
    agg_steps = 8 if schedule == "p-smem" else -(-len(pieces) // 2)
    k_steps = macs = a_bytes = w_bytes = 0
    per_chain = []
    for src, taps, n, ks in chains:
        c_steps = c_macs = 0
        for tidx in range(T):
            for ty in range(tiles_y):
                y0, y1 = ty * th, ty * th + th - 1
                for tx in range(tiles_x):
                    x0, x1 = tx * tw, tx * tw + tw - 1
                    for (dt, dy, dx), g in tap_groups(taps):
                        tt = tidx + dt
                        if tt < 0 or tt >= T or y1 + dy + g - 1 < 0 or y0 + dy >= H or x1 + dx < 0 or x0 + dx >= W:
                            continue
                        a_bytes += a_stage
                        w_bytes += g * 2 * n * 128
                        c_steps += g * ks
                        c_macs += g * ks * 3 * m * n * 16
        per_chain.append({"n": n, "k_steps_per_tap": ks, "taps": len(taps), "executed_k_steps": B * c_steps})
        k_steps += c_steps
        macs += c_macs
    n_tiles = T * tiles_x * tiles_y
    k_steps += n_tiles * agg_steps
    macs += n_tiles * agg_steps * 3 * m * 64 * 16
    if schedule == "p-smem":
        w_bytes += n_tiles * 2 * (2 * 64 * 128)
    if pb.res is not None:
        ks = (pb.res[6] - pb.res[5]) // 16
        k_steps += n_tiles * ks
        macs += n_tiles * ks * 3 * m * 64 * 16
        w_bytes += n_tiles * 2 * 64 * 128
        if schedule == "p-smem":
            a_bytes += n_tiles * a_stage
    a_bytes, w_bytes, k_steps, macs = B * a_bytes, B * w_bytes, B * k_steps, B * macs
    if schedule == "p-regs":
        w_bytes += min(B * n_tiles, n_sm) * 2 * (2 * 64 * 128)
    return {"tiles": B * n_tiles, "chains": per_chain, "agg_k_steps_per_tile": agg_steps, "executed_k_steps": k_steps,
            "macs": macs, "l2_act_bytes": a_bytes, "l2_weight_bytes": w_bytes, "l2_bytes": a_bytes + w_bytes}


def count_all(tm, th, tw, n_sm):
    blocks = {"block1": tm.model[0].packed()["tail"], "block2": tm.model[1].packed()["tail"]}
    return {s: {k: count_block(pb, s, th, tw, n_sm) for k, pb in blocks.items()} for s in SCHEDULES}


def capture_launches(tm, dev):
    """Runs the temporal model once and records the arguments of its two stp3_block_fused_fwd launches."""
    import torch
    from oracle.make_golden_dense import dense_input
    from stp3_b200 import dense
    calls = []
    orig = dense.block_tail

    def rec(*a, **k):
        calls.append((a, k))
        return orig(*a, **k)
    x = dense_input((B, T, 64 + N_CONST, H, W), 41)
    x[:, :, 64:] = x[:, :, 64:, :1, :1]
    dense.block_tail = rec
    try:
        with torch.no_grad():
            const = x[:, :, 64:, 0, 0].reshape(B * T, N_CONST).contiguous().to(dev)
            tm.forward_hl(dense.from_f32(x[:, :, :64].contiguous().to(dev)), const=const)
        torch.cuda.synchronize()
    finally:
        dense.block_tail = orig
    assert len(calls) == 2, "both blocks must take the back-to-back path"
    return calls


def time_blocks(args, tm):
    import torch
    from stp3_b200 import dense
    dev = torch.device("cuda:0")
    calls = capture_launches(tm, dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    outs = [None, None]

    def launch(i):
        a, k = calls[i]
        outs[i] = dense.block_tail(*a, **k)

    with torch.no_grad():
        for _ in range(args.warmup):
            launch(0); launch(1)
        torch.cuda.synchronize()
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.reps)]
        with ClockSampler() as clk:
            for e in ev:
                flush.zero_()                               # L2 evicted between repetitions, as bench.py does
                e[0].record(); launch(0); e[1].record(); launch(1); e[2].record()
            torch.cuda.synchronize()
        launch(0); launch(1)
        torch.cuda.synchronize()
    ms = {"block1": statistics.median(e[0].elapsed_time(e[1]) for e in ev),
          "block2": statistics.median(e[1].elapsed_time(e[2]) for e in ev)}
    res = {}
    for i, k in enumerate(("block1", "block2")):
        res[f"{k}_hi"] = outs[i].hi.cpu()
        res[f"{k}_lo"] = outs[i].lo.cpu()
        cs = calls[i][1].get("col_sums")
        if cs is not None:
            res[f"{k}_col_sums"] = cs.cpu()
    return ms, clk.mhz, torch.cuda.get_device_properties(0).multi_processor_count, res


def compare(res, ref_dir):
    import torch
    ref = torch.load(os.path.join(ref_dir, "block_outputs.pt"))
    out = {}
    for k, v in res.items():
        r = ref[k]
        if k.endswith("_col_sums"):
            out[k + "_max_rel"] = float(((v - r).abs().max() / r.abs().max().clamp_min(1e-30)).item())
        else:
            out[k + "_bitwise_equal"] = bool(torch.equal(v, r))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--tile", default="8x16", help="TH x TW pixels per CTA tile of the build being timed")
    ap.add_argument("--schedule", default="p-regs", choices=SCHEDULES, help="schedule of the build being timed")
    ap.add_argument("--sms", type=int, default=132, help="SM count for --count-only")
    ap.add_argument("--count-only", action="store_true")
    ap.add_argument("--save", metavar="DIR", help="torch.save both launches' hi / lo outputs and column sums")
    ap.add_argument("--compare", metavar="DIR", help="compare with the outputs another build saved with --save")
    args = ap.parse_args()
    th, tw = (int(v) for v in args.tile.split("x"))
    tm_cpu = build_model("cpu")
    line = {"shape": [B, T, 64 + N_CONST, H, W], "tile": args.tile, "schedule": args.schedule}
    if args.count_only:
        line["schedules"] = count_all(tm_cpu, th, tw, args.sms)
        print(json.dumps(line))
        return
    if args.reps < 50:
        ap.error("--reps must be >= 50")
    import torch
    tm = build_model("cuda:0")
    ms, mhz, n_sm, res = time_blocks(args, tm)
    counts = count_all(tm_cpu, th, tw, n_sm)
    line["schedules"] = counts
    line.update(gpu_info())
    line.update({"sm_mhz_during": mhz, "sms": n_sm, "reps": args.reps, "ms": ms, "ms_total": ms["block1"] + ms["block2"]})
    for k in ("block1", "block2"):
        c = counts[args.schedule][k]
        bound = c["macs"] * 2 / FLOP_PER_CLK_SM / (n_sm * mhz * 1e6) * 1e3 if mhz else None
        line[k] = {"ms": ms[k], "executed_k_steps": c["executed_k_steps"], "tensor_bound_ms": bound,
                   "tensor_bound_fraction": bound / ms[k] if bound else None, "l2_bytes": c["l2_bytes"],
                   "l2_tb_per_s": c["l2_bytes"] / (ms[k] * 1e-3) / 1e12}
    line["outputs"] = {k: int(v.view(torch.int16).long().sum().item()) if v.dtype == torch.bfloat16 else float(v.sum())
                       for k, v in res.items()}
    if args.save:
        os.makedirs(args.save, exist_ok=True)
        torch.save(res, os.path.join(args.save, "block_outputs.pt"))
    if args.compare:
        line["compare"] = compare(res, args.compare)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
