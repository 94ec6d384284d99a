"""Times the native EfficientNet-b4 trunk (cut after block 21) at the perceive shape -- B = 4 samples x 3 frames x 6
cameras = 72 images of 224x480 -- per stage and in total, against torch eager on the fp32 restatement of the same trunk
(oracle/efficientnet_oracle.py; cuDNN, TF32 off, channels_last, cudnn.benchmark) and with fp16 autocast, then the full
perceive step from images (GraphedPerception(entry="images")) in frames/s.

CUDA events; the L2 is flushed (256 MiB write) before every timed call; the variants alternate within each repetition;
the SM clock is sampled with nvidia-smi during the timed region.  Prints one JSON object.  Separate from bench.py's
contract line, which excludes the trunk on both arms.

    python tools/trunk_bench.py [--reps 10] [--batch 4]
"""
import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def stage_costs(nat, M, H, W):
    """Algorithmic FLOPs (2*MAC of the fp32 layers) and bytes (4 bytes per fp32 value: one bf16 hi/lo pair) per stage."""
    from stp3_b200 import dense
    from stp3_b200.models import efficientnet as EN
    c = {k: {"flops": 0.0, "bytes": 0.0} for k in ("stem", "expand", "depthwise", "se_gate", "project")}
    h, w = EN.out_size(H, 3, 2, nat.stem_pad), EN.out_size(W, 3, 2, nat.stem_pad)
    stem = nat._conv_stem.out_channels
    c["stem"]["flops"] += 2.0 * M * h * w * stem * 27
    c["stem"]["bytes"] += 4.0 * M * (3 * H * W + h * w * dense.pad_to(stem))
    for blk in nat._blocks:
        s = blk.spec
        px_in = M * h * w
        if s.exp != s.cin:
            c["expand"]["flops"] += 2.0 * px_in * s.cin * s.exp
            c["expand"]["bytes"] += 4.0 * px_in * (dense.pad_to(s.cin) + dense.pad_to(s.exp))
        h, w = EN.out_size(h, s.k, s.stride, s.pad), EN.out_size(w, s.k, s.stride, s.pad)
        px = M * h * w
        c["depthwise"]["flops"] += 2.0 * px * s.exp * s.k * s.k
        c["depthwise"]["bytes"] += 4.0 * (px_in + px) * dense.pad_to(s.exp)
        elems = dense.se_proj_weight_elems(s.exp, s.cout)
        c["se_gate"]["flops"] += 2.0 * M * (2 * s.exp * s.se + s.exp * s.cout)
        c["se_gate"]["bytes"] += 2.0 * M * elems + 4.0 * s.cout * s.exp
        c["project"]["flops"] += 2.0 * px * s.exp * s.cout
        c["project"]["bytes"] += 4.0 * px * (dense.pad_to(s.exp) + dense.pad_to(s.cout) * (2 if s.skip else 1)) + 2.0 * M * elems
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4)
    args = ap.parse_args()

    import torch
    import bench
    from oracle import efficientnet_oracle as EO
    from stp3_b200.models.stp3 import GraphedPerception
    from stp3_b200.utils import synthetic as syn

    if not torch.cuda.is_available():
        raise SystemExit("trunk_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    S, N = 3, 6
    M, H, W = args.batch * S * N, 224, 480

    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=0), 'b4').eval()
    model = bench.build_model(None)
    from stp3_b200.models.encoder import Encoder
    enc = model.encoder
    model.encoder = Encoder(model.cfg.MODEL.ENCODER, model.depth_channels, backbone="native")
    model.encoder.load_state_dict({**{f"backbone.{k}": v for k, v in ora.state_dict().items()},
                                   **{k: v for k, v in enc.state_dict().items() if not k.startswith("backbone.")}},
                                  strict=True)
    model = model.eval().to(dev)
    nat = model.encoder.backbone
    torch_fp32 = copy.deepcopy(ora).to(dev).to(memory_format=torch.channels_last)

    torch.manual_seed(0)
    x = torch.randn(M, 3, H, W, device=dev)
    x_cl = x.contiguous(memory_format=torch.channels_last)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def native():
        return nat.forward_hl(x)

    def eager_fp32():
        return EO.endpoints(torch_fp32, x_cl)

    def eager_fp16():
        with torch.autocast("cuda", dtype=torch.float16):
            return EO.endpoints(torch_fp32, x_cl)

    variants = {"native": native, "torch_fp32_cudnn": eager_fp32, "torch_fp16_autocast": eager_fp16}
    with torch.no_grad():
        for fn in variants.values():          # warm-up: packing, autotuning, cuDNN algorithm search
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        # the native trunk as one CUDA graph (how GraphedPerception runs it): device time without the host cost of
        # ~215 eager launches
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            native()
        variants["native_graphed"] = graph.replay
        # parity of the timed native call against the fp32 restatement (same inputs)
        r3, r4 = nat(x)
        o3, o4 = eager_fp32()
        parity = {n: ((a - b).abs().max() / b.abs().max()).item() for n, a, b in (("reduction_3", r3, o3), ("reduction_4", r4, o4))}

        clocks = bench.ClockSampler(0)
        clocks.start()
        times = {k: [] for k in variants}
        stage_ms = {}
        for _ in range(args.reps):
            for name, fn in variants.items():
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b))
        # per stage (a separate pass: the marks add an event record between launches)
        for _ in range(args.reps):
            flush.zero_()
            nat.stage_events = []
            native()
            torch.cuda.synchronize()
            ev = nat.stage_events
            nat.stage_events = None
            acc = {}
            for (_, e0), (name, e1) in zip(ev, ev[1:]):
                acc[name] = acc.get(name, 0.0) + e0.elapsed_time(e1)
            for k, v in acc.items():
                stage_ms.setdefault(k, []).append(v)
        clk = clocks.stop()

        # the full perceive step from images, one CUDA graph
        inp = syn.lift_inputs(syn.CONFIGS["perceive"], args.batch, seed=0, random_pose=False)
        image = torch.randn(args.batch, S, N, 3, H, W)
        g = GraphedPerception(model, args.batch, N, dev, entry="images")
        g.stage_inputs(image, None, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        for _ in range(3):
            g.graph.replay()
        torch.cuda.synchronize()
        step = []
        for _ in range(args.reps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.graph.replay()
            b.record()
            b.synchronize()
            step.append(a.elapsed_time(b))

    pk = bench.peaks()
    costs = stage_costs(nat, M, H, W)
    stages = {}
    for k, c in costs.items():
        ms = statistics.median(stage_ms[k])
        e = {"ms": ms, "gflop": c["flops"] / 1e9, "mbytes": c["bytes"] / 1e6,
             "hbm_frac": c["bytes"] / (ms * 1e-3) / (pk["hbm_gbs"] * 1e9)}
        if k in ("expand", "project", "stem"):
            e["tensor_frac"] = c["flops"] / (ms * 1e-3) / (pk["bf16_tflops"] * 1e12)
        stages[k] = e
    med = {k: statistics.median(v) for k, v in times.items()}
    gpu = os.popen("nvidia-smi --query-gpu=name,power.limit --format=csv,noheader -i 0").read().strip()
    print(json.dumps({
        "what": "EfficientNet-b4 trunk (blocks 0-21), perceive shape", "images": M, "image_hw": [H, W],
        "gpu": gpu, "clocks": clk, "peaks": pk,
        "algorithmic_gflop": sum(c["flops"] for c in costs.values()) / 1e9,
        "ms_median": med, "ms_all": times,
        "native_graphed_vs_torch_fp32": med["torch_fp32_cudnn"] / med["native_graphed"],
        "native_graphed_vs_torch_fp16": med["torch_fp16_autocast"] / med["native_graphed"],
        "native_stages": stages, "native_launches": 1 + sum(nat.launches_per_block()),
        "parity_native_vs_fp32_restatement": parity,
        "perceive_step_from_images": {"ms_median": statistics.median(step), "frames_per_s": args.batch / (statistics.median(step) * 1e-3),
                                      "how": "GraphedPerception(entry='images') replay, L2 flushed before each"},
    }, indent=1))


if __name__ == "__main__":
    main()
