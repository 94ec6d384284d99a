"""Device time of the DeepLab head's two back-to-back launches (stp3_aspp_fused_fwd: the ASPP instance = four branches
+ projection, the tail instance = 3x3 conv + classifier) at the perceive shape (B=4, T=3, 64 x 200 x 200, hidden 128),
set against what the tile schedule asks of the tensor pipe and of L2.

    python tools/head_bench.py [--reps 100] [--warmup 10] [--cluster C] [--group GYxGX]
    python tools/head_bench.py --count-only            # the host-side step / byte counts, no GPU
    python tools/head_bench.py --profile-step DIR      # per-kernel device time of one replayed perceive step

The counts restate aspp_fused.cu's schedule on the host: one CTA per 8 x 16 tile (group 1x1), a tap skipped when it is
padding for the tile, each executed K step moving one 32 KB activation stage and one 32 KB weight stage from L2.  The
other groupings are what a thread-block-cluster schedule would do: a cluster of C = GY x GX CTAs takes GY x GX
neighbouring tiles in lockstep, skips a tap only when it is padding for every tile of the group, and reads each weight
stage from L2 once per group (TMA multicast).  --cluster / --group name the schedule of the build being timed.  One
JSON line with the GPU name, power limit and the SM clock sampled during the timed loop (DESIGN.md 3.4).
"""
import argparse
import csv
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGE_BYTES = 32 * 1024            # one activation stage (hi + lo, 128 pixels x 64 ch) = one weight stage (hi + lo, 128 x 64)
FLOP_PER_STEP = 2 * 12 * 2 * 64 * 128 * 16      # 2 warpgroups x 12 wgmma.m64n128k16
FLOP_PER_CLK_SM = 4096                          # dense bf16 wgmma rate of one H100 SM
B, T, H, W = 4, 3, 200, 200
RATES = (12, 24, 36)


def head_taps():
    """(taps per branch, kblocks) of the two instances, in the order DeepLabHead._pack hands them to the kernel."""
    def taps3(d):
        return [((iy - 1) * d, (ix - 1) * d) for iy in range(3) for ix in range(3)]
    aspp = [[(0, 0)]] + [taps3(r) for r in RATES]
    tail = [taps3(1)]
    return {"aspp": (aspp, 1), "tail": (tail, 2)}


def count_schedule(branches, kblocks, n_img, h, w, gy, gx):
    """Host restatement of the head's tile schedule for groups of gy x gx tiles (1 x 1: aspp_fused.cu).  Returns the K steps the tensor
    cores execute (tiles x steps), the step slots the clusters occupy (groups x steps x cluster size) and the operand
    bytes every CTA pulls from L2 (activations per tile, weights once per group)."""
    tiles_x, tiles_y = -(-w // 16), -(-h // 8)
    groups_x, groups_y = -(-tiles_x // gx), -(-tiles_y // gy)
    c = gy * gx
    n_br = len(branches)
    mma = slots = a_bytes = w_bytes = 0
    for gyi in range(groups_y):
        ty1 = min((gyi + 1) * gy, tiles_y)
        y0, y1 = gyi * gy * 8, ty1 * 8 - 1
        for gxi in range(groups_x):
            tx1 = min((gxi + 1) * gx, tiles_x)
            x0, x1 = gxi * gx * 16, tx1 * 16 - 1
            n_tiles = (ty1 - gyi * gy) * (tx1 - gxi * gx)
            steps = 0
            for taps in branches:
                for dy, dx in taps:
                    if y1 + dy < 0 or y0 + dy >= h or x1 + dx < 0 or x0 + dx >= w:
                        continue                       # padding for every tile of the group
                    steps += kblocks
            proj = 2 * n_br
            mma += n_tiles * (steps + proj)
            slots += c * (steps + proj)
            a_bytes += n_tiles * steps * STAGE_BYTES
            w_bytes += (steps + proj) * STAGE_BYTES
    n = n_img
    return {"tiles": n * tiles_x * tiles_y, "groups": n * groups_x * groups_y, "mma_k_steps": n * mma,
            "occupied_k_step_slots": n * slots, "l2_act_bytes": n * a_bytes, "l2_weight_bytes": n * w_bytes,
            "l2_bytes": n * (a_bytes + w_bytes)}


def schedules(gy, gx):
    return {k: count_schedule(br, kb, B * T, H, W, gy, gx) for k, (br, kb) in head_taps().items()}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power, mx = [f.strip() for f in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(power), "sm_max_mhz": float(mx)}
    except Exception as e:                              # noqa: BLE001  (reported as unknown)
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None, "nvidia_smi_error": str(e)}


class ClockSampler:
    """nvidia-smi SM clock every 100 ms while the timed loop runs."""

    def __enter__(self):
        fd, self.path = tempfile.mkstemp(suffix=".csv")
        os.close(fd)
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", "0"], stdout=open(self.path, "w"),
                                         stderr=subprocess.DEVNULL)
        except Exception:                               # noqa: BLE001
            self.proc = None
        return self

    def __exit__(self, *exc):
        self.mhz = None
        if self.proc is not None:
            time.sleep(0.15)
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:                           # noqa: BLE001
                self.proc.kill()
                self.proc.wait()
            vals = []
            for line in open(self.path):
                try:
                    vals.append(float(line.strip()))
                except ValueError:
                    pass
            self.mhz = statistics.median(vals) if vals else None
        os.unlink(self.path)


def time_head(args):
    import torch
    from oracle import torch_dense as TD
    from stp3_b200 import dense
    from stp3_b200.layers.convolutions import DeepLabHead

    dev = torch.device("cuda:0")
    with torch.no_grad():
        head = TD.init_exact(DeepLabHead(64, 64, hidden_channel=128), seed=17).eval().to(dev)
        P = head.packed()
        assert "fused" in P and "tail" in P, "the head must take the back-to-back path"
        x = dense.from_f32(TD.exact_gauss((B, T, 64, H, W), torch.Generator().manual_seed(18)).to(dev))
        pbias = TD.exact_gauss((B * T, 128), torch.Generator().manual_seed(19)).to(dev).contiguous()
        tbias = P["tail"].proj_bias.unsqueeze(0).expand(B * T, -1).contiguous()
        mid = dense.HL.empty(B, T, H, W, 128, dev, cp=128)
        out = dense.HL.empty(B, T, H, W, 64, dev, cp=64)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def aspp():
        dense.aspp_fused(x, P["fused"], pbias, out=mid)

    def tail():
        dense.aspp_fused(mid, P["tail"], tbias, out=out, relu=False, n_store=64)

    for _ in range(args.warmup):
        aspp(); tail()
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.reps)]
    with ClockSampler() as clk:
        for e in ev:
            flush.zero_()                               # L2 evicted between repetitions, as bench.py does
            e[0].record(); aspp(); e[1].record(); tail(); e[2].record()
        torch.cuda.synchronize()
    ms_aspp = statistics.median(e[0].elapsed_time(e[1]) for e in ev)
    ms_tail = statistics.median(e[1].elapsed_time(e[2]) for e in ev)
    # outputs of one more call, hashed: two builds with the same schedule semantics must agree bitwise
    aspp(); tail()
    torch.cuda.synchronize()
    digest = {"mid_hi_sum": int(mid.hi.view(torch.int16).long().sum().item()),
              "out_hi_sum": int(out.hi.view(torch.int16).long().sum().item()),
              "out_lo_sum": int(out.lo.view(torch.int16).long().sum().item())}
    if args.save_outputs:                           # for a bitwise comparison of two builds
        torch.save({k: t.cpu() for k, t in (("mid_hi", mid.hi), ("mid_lo", mid.lo), ("out_hi", out.hi),
                                             ("out_lo", out.lo))}, args.save_outputs)
    return {"aspp": ms_aspp, "tail": ms_tail}, clk.mhz, torch.cuda.get_device_properties(0).multi_processor_count, digest


def profile_step(out_dir):
    """Per-kernel device time of ONE replayed step of the graphed perceive workload (bench.py's step), from
    torch.profiler CUDA activity, written to out_dir/perceive_step_kernels.csv."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from stp3_b200.models.stp3 import GraphedPerception
    from stp3_b200.utils import synthetic as syn

    cfg = syn.CONFIGS["perceive"]
    dev = torch.device("cuda:0")
    b = 4
    prob = bench.make_problem(cfg, b, seed=0)
    inp = prob["inp"]
    model = bench.build_model(dev, cfg)
    with torch.no_grad():
        g = GraphedPerception(model, b, cfg.n_cameras, dev, entry="lift")
        g(inp["feat"].to(dev), inp["depth_logits"].to(dev), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        for _ in range(5):
            g.graph.replay()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g.graph.replay()
            torch.cuda.synchronize()
    rows = []
    for e in prof.events():
        t = float(getattr(e, "device_time", 0.0) or getattr(e, "cuda_time", 0.0) or 0.0)
        if t > 0:
            rows.append((e.name, t))
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "perceive_step_kernels.csv"), "w", newline="") as f:
        wr = csv.writer(f)
        wr.writerow(["kernel", "device_us"])
        for r in rows:
            wr.writerow(r)
    total = sum(t for _, t in rows)
    by = {}
    for n, t in rows:
        k = n.split("(")[0].split("<")[0].strip()
        by[k] = by.get(k, 0.0) + t
    head = sum(t for n, t in rows if "aspp_fused" in n)
    print(json.dumps({**gpu_info(), "step_kernel_us": round(total, 1), "aspp_fused_us": round(head, 1),
                      "aspp_fused_share": round(head / total, 4) if total else None,
                      "by_kernel_us": {k: round(v, 1) for k, v in sorted(by.items(), key=lambda kv: -kv[1])}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cluster", type=int, default=1, help="cluster size of the build being timed")
    ap.add_argument("--group", default="1x1", help="GYxGX tiles per cluster of the build being timed")
    ap.add_argument("--count-only", action="store_true")
    ap.add_argument("--save-outputs", metavar="FILE", help="torch.save both launches' hi / lo output planes")
    ap.add_argument("--profile-step", metavar="DIR")
    args = ap.parse_args()
    if args.profile_step:
        profile_step(args.profile_step)
        return
    gy, gx = (int(v) for v in args.group.split("x"))
    assert gy * gx == args.cluster, "--group must hold --cluster tiles"
    counts = {f"{a}x{b}": schedules(a, b) for a, b in ((1, 1), (2, 1), (1, 2), (4, 1), (2, 2))}
    line = {"shape": [B, T, 64, H, W], "cluster": args.cluster, "group": args.group, "schedules": counts}
    if not args.count_only:
        if args.reps < 50:
            ap.error("--reps must be >= 50")
        ms, mhz, n_sm, digest = time_head(args)
        line.update(gpu_info())
        line.update({"sm_mhz_during": mhz, "sms": n_sm, "reps": args.reps, "ms": ms, "ms_total": ms["aspp"] + ms["tail"],
                     "outputs": digest})
        own = counts[args.group]
        for k in ("aspp", "tail"):
            c = own[k]
            bound = (c["mma_k_steps"] * FLOP_PER_STEP / FLOP_PER_CLK_SM / (n_sm * mhz * 1e6) * 1e3) if mhz else None
            line[k] = {"ms": ms[k], "mma_k_steps": c["mma_k_steps"], "tensor_bound_ms": bound,
                       "tensor_bound_fraction": (bound / ms[k]) if bound else None,
                       "l2_bytes": c["l2_bytes"], "l2_tb_per_s": c["l2_bytes"] / (ms[k] * 1e-3) / 1e12}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
