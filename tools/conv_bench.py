"""Device time of every implicit-GEMM convolution (stp3_conv_fwd) of one perceive step (B = 4, seeded as bench.py
builds the model): the temporal model's and the decoder's calls of one eval forward_hl, and with --heads the encoder
heads' calls first.  Each recorded call is replayed alone under the tiling the autotuner chose for it, as a CUDA graph,
with L2 flushed before every repetition.  Per layer: taps x Cin -> Cout, output map, tiles, microseconds and the
tensor-bound fraction (3 bf16 products per MAC at the data-sheet rate, scaled to the SM clock sampled during the
timed loop), and the HBM traffic the call cannot avoid (input window read once, every output stored once) over its
time.

    python tools/conv_bench.py [--heads] [--reps 100] [--blocks 128|64s|64p] [--save DIR | --compare DIR] [--lib PATH]
    python tools/conv_bench.py --count-only [--sms 132]     # host counts of the decoder's 25x25 / 50x50 layers, no GPU

--save DIR writes the tilings and a SHA-256 digest of every output of every call (hi / lo planes, second destination,
fp32 outputs, fused-head planes, column sums, each snapshotted right after its call); --compare DIR runs under the
tilings another build saved there and reports which outputs are not bitwise identical.  --lib loads another build of
libstp3_b200.so, so that two builds can be timed alternately on the same card.  --blocks replaces the tuner's
column-block choice for every convolution of 128 / 256 columns that may run in blocks (128-column blocks, 64-column
stacked, 64-column plain), so each width is timed alone.  --count-only prints, for the decoder trunk's low-resolution
layers under each block width, what stp3_conv_tiling answers: work items, waves over the SMs, ring depths.  One JSON line.
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
BLOCKS = {"128": 0, "64s": 16 + 8, "64p": 16}        # group bits of dense.conv's tune
# (taps, cin, cout, stride, input map, output map) of the decoder trunk's calls on the 25 x 25 and 50 x 50 maps of one
# perceive step (ResNet-18 layer2 / layer3 and the 1x1 of the two upsampling stages), B * T = 12 images
LOW_RES_LAYERS = [(9, 128, 256, 2, 50, 25), (1, 128, 256, 2, 50, 25)] + [(9, 256, 256, 1, 25, 25)] * 3 + \
                 [(1, 256, 128, 1, 25, 25), (9, 64, 128, 2, 100, 50), (1, 64, 128, 2, 100, 50)] + \
                 [(9, 128, 128, 1, 50, 50)] * 3 + [(1, 128, 64, 1, 50, 50)]


def count_layers(n_sm, n_img=3 * BATCH):
    """stp3_conv_tiling of every LOW_RES_LAYERS entry under each column-block width (host arithmetic only)."""
    import ctypes
    import torch
    from stp3_b200 import _lib, dense
    rows = []
    for taps, cin, cout, stride, hw_in, hw_out in LOW_RES_LAYERS:
        k = 3 if taps == 9 else 1
        pc = dense.pack_conv(torch.zeros(cout, cin, k, k), torch.zeros(cout), stride=stride)
        d = _lib.ConvDesc(B=n_img, T=1, H=hw_in, W=hw_in, in_cstride=cin, cin=cin, Ho=hw_out, Wo=hw_out, stride=stride,
                          ntaps=taps, bn=pc.bn)
        for i, t in enumerate(pc.taps):
            d.taps[i][0], d.taps[i][1], d.taps[i][2] = t
        row = {"layer": f"{taps}x{cin}->{cout}" + (f" s{stride}" if stride > 1 else ""), "map": f"{n_img}x{hw_out}x{hw_out}"}
        for name, bits in BLOCKS.items():
            if pc.bn < 128 and name != "128":
                continue
            d.tune_group, d.tune_bn = bits & 15, 64 if bits & dense.BLOCKS64 else 0
            info = _lib.ConvTilingInfo()
            _lib.check(_lib.lib().stp3_conv_tiling(ctypes.byref(d), n_sm, ctypes.byref(info)), "stp3_conv_tiling")
            row[name] = {"items": info.items, "waves": round(info.items / n_sm, 2), "a_stages": info.a_stages,
                         "b_stages": info.b_stages, "resident": bool(info.resident)}
        rows.append(row)
    return rows


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
        seen.append(d._obj.tune_group | (dense.BLOCKS64 if d._obj.tune_bn == 64 else 0))
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
    # bytes: hi + lo bf16 (4 B) per channel of the input frames the taps reach and of every stored output channel
    frames_in = min(x.hi.shape[1], T + max(0, -min(t[0] for t in pc.taps)))
    stored = 0
    if k.get("store", True) and (k.get("out") is not None or k.get("out_f32") is None and k.get("head") is None):
        stored += 4 * (k.get("n_store") or pc.bn)
    if k.get("out2") is not None:
        stored += 4 * (k.get("n_store2") or 64)
    if k.get("out_f32") is not None:
        stored += 4 * k["n_valid"]
    if k.get("head") is not None:
        stored += 4 * len(k["head"]["outs"])
    nbytes = B * frames_in * H * W * pc.cin_p * 4 + n_img * Ho * Wo * stored
    return {"layer": f"{len(pc.taps)}x{cin}->{pc.cout}" + (f" s{pc.stride}" if pc.stride > 1 else ""),
            "map": f"{n_img}x{Ho}x{Wo}", "tiles": n_img * -(-Ho // 8) * -(-Wo // 16), "flop": 3 * 2 * macs,
            "bytes": nbytes}


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
    ap.add_argument("--blocks", choices=list(BLOCKS), help="column blocks of every 128 / 256-column convolution")
    ap.add_argument("--count-only", action="store_true", help="host counts of the low-resolution decoder layers")
    ap.add_argument("--sms", type=int, default=132, help="SM count for --count-only")
    args = ap.parse_args()
    if args.count_only:
        print(json.dumps({"sms": args.sms, "layers": count_layers(args.sms)}))
        return
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
    if args.blocks:      # the tuned tap sharing of every call, the column blocks as asked
        def in_blocks(a, k):
            return a[1].bn >= 128 and k.get("head") is None and k.get("out2") is None
        calls = record_step(model, dev, args.heads, [(t & 3) | BLOCKS[args.blocks] if in_blocks(a, k) else t
                                                     for a, k, t, _ in calls])
    us, mhz = time_calls(calls, args.reps, dev)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    rows, saved = [], []
    for i, ((a, k, tiling, dig), t) in enumerate(zip(calls, us)):
        info = layer_info(a, k)
        bound_us = info["flop"] / (FLOP_PER_CLK_SM * n_sm * mhz * 1e6) * 1e6 if mhz else None
        row = dict(i=i, **info, tiling=tiling, us=round(t, 2), gb_per_s=round(info["bytes"] / (t * 1e3), 1),
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
