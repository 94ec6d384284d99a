"""Device time of every implicit-GEMM convolution (stp3_conv_fwd) of one perceive step (B = 4, seeded as bench.py
builds the model): the temporal model's and the decoder's calls of one eval forward_hl, and with --heads the encoder
heads' calls first.  Each recorded call is replayed alone under the tiling the autotuner chose for it, as a CUDA graph,
with L2 flushed before every repetition.  Per layer: taps x Cin -> Cout, output map, tiles, microseconds and the
tensor-bound fraction (3 bf16 products per MAC at the data-sheet rate, scaled to the SM clock sampled during the
timed loop).

    python tools/conv_bench.py [--heads] [--reps 100] [--save DIR | --compare DIR] [--lib PATH]

--save DIR writes the tilings and a SHA-256 digest of every output of every call (hi / lo planes, second destination,
fp32 outputs, fused-head planes, column sums, each snapshotted right after its call); --compare DIR runs under the
tilings another build saved there and reports which outputs are not bitwise identical.  --lib loads another build of
libstp3_b200.so, so that two builds can be timed alternately on the same card.  One JSON line.
"""
import argparse
import hashlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from head_bench import FLOP_PER_CLK_SM, ClockSampler, gpu_info  # noqa: E402

BATCH = 4


def outputs_of(a, k, ret):
    """What one dense.conv call wrote: name -> tensor (the channel window of a destination it shares with other calls)."""
    out = {}
    pc = a[1]
    hl = ret if ret is not None else k.get("out")
    if hl is not None:
        c0 = k.get("out_coff", 0)
        c1 = c0 + (k.get("n_store") or pc.bn)
        out["hi"], out["lo"] = hl.hi[..., c0:c1], hl.lo[..., c0:c1]
    if k.get("out2") is not None:
        c0 = k.get("out2_coff", 0)
        c1 = c0 + (k.get("n_store2") or 64)
        out["out2_hi"], out["out2_lo"] = k["out2"].hi[..., c0:c1], k["out2"].lo[..., c0:c1]
    if k.get("out_f32") is not None:
        out["f32"] = k["out_f32"]
    if k.get("head") is not None:
        for i, (t, ch) in enumerate(k["head"]["outs"]):
            out[f"head{i}"] = t[:, ch]
    if k.get("col_sums") is not None:
        out["col_sums"] = k["col_sums"]
    return out


def digest(t):
    import torch
    return hashlib.sha256(t.detach().contiguous().cpu().view(-1).view(torch.uint8).numpy()).hexdigest()


def record_step(model, dev, heads, tilings):
    """One eval step with dense.conv wrapped: returns [(args, kwargs, tiling, {output: digest})] in call order.  The
    tiling of each launch is read from the descriptor it passes; `tilings` (a list, or None) forces them instead."""
    import torch
    import bench
    from stp3_b200 import _lib, dense
    from stp3_b200.utils import synthetic as syn
    cfg = syn.CONFIGS["perceive"]
    S, C = cfg.receptive_field, model.encoder_out_channels
    X, Y = model.bev_size
    prob = bench.make_problem(cfg, BATCH, seed=0)
    h = model.prepare_inputs(prob["inp"]["intrinsics"], prob["inp"]["extrinsics"], prob["inp"]["future_egomotion"])
    const = h["const"].to(dev)
    bev = dense.from_f32(syn.exact_gauss((BATCH, S, C, X, Y), torch.Generator().manual_seed(7)).to(dev))
    r_lo, r_hi = (t.to(dev) for t in bench.trunk_endpoints(cfg, BATCH, 0))

    def step():
        if heads:
            model.encoder.heads_f32(r_lo.flatten(0, 2), r_hi.flatten(0, 2), channels_last=True)
        model.decoder.forward_hl(model.temporal_model.forward_hl(bev, const=const))

    lib = _lib.lib()
    fwd = lib.stp3_conv_fwd
    seen = []

    def fwd_rec(d, *rest):
        seen.append(d._obj.tune_group)
        return fwd(d, *rest)

    calls = []
    orig = dense.conv

    def rec(*a, **k):
        if tilings is not None:
            k = dict(k, tune=(0, tilings[len(calls)]))
        n0 = len(seen)
        ret = orig(*a, **k)
        assert len(seen) == n0 + 1
        torch.cuda.synchronize()
        calls.append((a, dict(k, tune=(0, seen[-1])), seen[-1], {n: digest(t) for n, t in outputs_of(a, k, ret).items()}))
        return ret

    with torch.no_grad():
        step()                                   # autotunes every layer (or warms the forced tilings)
        torch.cuda.synchronize()
        dense.conv, lib.stp3_conv_fwd = rec, fwd_rec
        try:
            step()
        finally:
            dense.conv, lib.stp3_conv_fwd = orig, fwd
    return calls


def layer_info(a, k):
    x, pc = a[0], a[1]
    B, T, H, W, _ = x.hi.shape
    if k.get("frames") is not None:
        T = k["frames"][1]
    Ho, Wo = k.get("out_hw") or ((H + pc.stride - 1) // pc.stride, (W + pc.stride - 1) // pc.stride)
    n_img = B * T
    cin = (pc.k_hi - pc.k_lo) if pc.k_hi else pc.cin_p
    macs = n_img * Ho * Wo * len(pc.taps) * cin * pc.cout
    return {"layer": f"{len(pc.taps)}x{cin}->{pc.cout}" + (f" s{pc.stride}" if pc.stride > 1 else ""),
            "map": f"{n_img}x{Ho}x{Wo}", "tiles": n_img * -(-Ho // 8) * -(-Wo // 16), "flop": 3 * 2 * macs}


def time_calls(calls, reps, dev):
    import torch
    from stp3_b200 import dense
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    graphs = []
    with torch.no_grad():
        for a, k, _, _ in calls:
            dense.conv(*a, **k)                  # warm outside the capture
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                dense.conv(*a, **k)
            graphs.append(g)
        us = []
        with ClockSampler() as clk:
            for g in graphs:
                t = []
                for _ in range(reps):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); g.replay(); e1.record()
                    t.append((e0, e1))
                torch.cuda.synchronize()
                us.append(statistics.median(e0.elapsed_time(e1) * 1e3 for e0, e1 in t))
    return us, clk.mhz


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", action="store_true", help="also record the encoder heads' convolutions")
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--save", metavar="DIR", help="write the tilings and output digests of every call")
    ap.add_argument("--compare", metavar="DIR", help="run under the tilings saved in DIR and compare output digests")
    ap.add_argument("--lib", metavar="PATH", help="libstp3_b200.so to load instead of the package's own")
    args = ap.parse_args()
    import torch
    from stp3_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    import bench
    assert torch.cuda.is_available(), "conv_bench.py needs a CUDA device"
    dev = torch.device("cuda:0")
    ref = None
    if args.compare:
        with open(os.path.join(args.compare, "conv_outputs.json")) as f:
            ref = json.load(f)
        assert ref["heads"] == args.heads, "--compare needs the --heads setting of the saved run"
    model = bench.build_model(dev)
    calls = record_step(model, dev, args.heads, [c["tiling"] for c in ref["calls"]] if ref else None)
    us, mhz = time_calls(calls, args.reps, dev)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    rows, saved = [], []
    for i, ((a, k, tiling, dig), t) in enumerate(zip(calls, us)):
        info = layer_info(a, k)
        bound_us = info["flop"] / (FLOP_PER_CLK_SM * n_sm * mhz * 1e6) * 1e6 if mhz else None
        row = dict(i=i, **info, tiling=tiling, us=round(t, 2),
                   tensor_bound_fraction=round(bound_us / t, 3) if bound_us else None)
        if ref:
            r = ref["calls"][i]
            row["identical"] = r["digests"] == dig
            if not row["identical"]:
                row["differs"] = sorted(n for n in dig if r["digests"].get(n) != dig[n])
        rows.append(row)
        saved.append({"layer": info["layer"], "tiling": tiling, "digests": dig})
    line = {"lib": _lib.LIB_PATH, "heads": args.heads, **gpu_info(), "sm_mhz_during": mhz, "sms": n_sm,
            "reps": args.reps, "total_us": round(sum(us), 1), "layers": rows}
    if ref:
        assert len(ref["calls"]) == len(calls), "the saved run recorded a different number of calls"
        line["all_identical"] = all(r["identical"] for r in rows)
    if args.save:
        os.makedirs(args.save, exist_ok=True)
        with open(os.path.join(args.save, "conv_outputs.json"), "w") as f:
            json.dump({"heads": args.heads, "calls": saved}, f)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
