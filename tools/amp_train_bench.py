"""Train-step time of the train-mode modules in fp32 and under fp16 / bf16 autocast (the one-product convolutions),
alternated in one process: DeepLabHead, UpsamplingConcat (encoder head sizes), the Decoder and the TemporalModel at the
perceive size (B = 1, S = 3, 200 x 200 BEV), and the whole model behind the trunk at that size: STP3 in train mode
entered at precomputed trunk endpoints (6 cameras x 3 frames, 224 x 480 images): encoder heads, lift-splat,
TemporalModel and Decoder in one step.  One step = forward under the mode + backward outside
it.  Also reports the peak memory of a step, the per-kernel time of the convolution and weight-gradient kernels of the
Decoder, TemporalModel and whole-model steps in each mode (torch.profiler, a separate pass), and the GPU name, power limit and SM clock read in the
same run.  Prints one JSON line.

    python tools/amp_train_bench.py [--steps 10] [--warmup 3] [--rounds 3]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import torch_dense as TD  # noqa: E402
from stp3_b200.layers.convolutions import DeepLabHead, UpsamplingConcat  # noqa: E402
from stp3_b200.models.decoder import Decoder  # noqa: E402
from stp3_b200.models.temporal_model import TemporalModel  # noqa: E402

DEV = "cuda:0"
MODES = {"fp32": None, "fp16": torch.float16, "bf16": torch.bfloat16}
GATES = dict(perceive_hdmap=True, predict_pedestrian=True, predict_instance=False, predict_future_flow=False,
             planning=False)


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        p, sm, sm_max = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update(power_limit_w=float(p), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(sm_max))
    except Exception:                               # noqa: BLE001  (reported as unknown)
        info.update(power_limit_w=None, sm_clock_mhz=None)
    return info


def cases():
    g = torch.Generator().manual_seed(0)

    def rnd(*s):
        return TD.exact_gauss(s, g).to(DEV)
    head = TD.init_exact(DeepLabHead(160, 160, hidden_channel=64), seed=3).to(DEV).train()
    xh = rnd(18, 160, 14, 30)
    up = TD.init_exact(UpsamplingConcat(64 + 160, 64), seed=4).to(DEV).train()
    xu, xf = rnd(18, 160, 14, 30), rnd(18, 64, 28, 60)
    dec = TD.init_exact(Decoder(64, 2, 3, 2, GATES), seed=2).to(DEV).train()
    xd = rnd(1, 3, 64, 200, 200)
    tm = TD.init_exact(TemporalModel(70, 3, (200, 200), start_out_channels=64), seed=3).to(DEV).train()
    tm.model[0].n_const = 6
    xt, ct = rnd(1, 3, 64, 200, 200), rnd(3, 6)

    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    from stp3_b200.utils import synthetic as syn
    lcfg = syn.LiftSplatConfig()
    model = STP3(get_cfg(), backbone=torch.nn.Identity())
    with torch.no_grad():
        geo = {k: getattr(model, k).detach().clone() for k in ("frustum", "bev_resolution", "bev_start_position",
                                                               "bev_dimension")}
        TD.init_exact(model, seed=7)
        for k, v in geo.items():
            getattr(model, k).copy_(v)
    model = model.to(DEV).train()
    Hf, Wf = lcfg.feat_hw
    r_lo, r_hi = rnd(1, 3, 6, 56, Hf, Wf), rnd(1, 3, 6, 160, Hf // 2, Wf // 2)
    li = syn.lift_inputs(lcfg, 1, seed=4, random_pose=True)

    def loss(out):
        if isinstance(out, dict):
            return sum(v.float().square().mean() for v in out.values() if v is not None)
        return out.float().square().mean()
    return {"deeplab_head_18x14x30": (head, lambda: loss(head(xh))),
            "upsampling_concat_18x28x60": (up, lambda: loss(up(xu, xf))),
            "decoder_1x3x200x200": (dec, lambda: loss(dec(xd))),
            "temporal_model_1x3x200x200": (tm, lambda: loss(tm(xt, const=ct))),
            "stp3_behind_trunk_6x3_200x200": (model, lambda: loss(model.forward_trunk_features(
                r_lo, r_hi, li["intrinsics"], li["extrinsics"], li["future_egomotion"])))}


def step(mod, fwd, mode):
    mod.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=mode or torch.float16, enabled=mode is not None):
        loss = fwd()
    loss.backward()


def timed(mod, fwd, mode, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step(mod, fwd, mode)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def kernel_times(mod, fwd, mode):
    """mean device time per launch of the convolution / weight-gradient kernels in one step (us)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(mod, fwd, mode)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        n = e.key
        if "conv_igemm_kernel" in n or "wgrad_partial_kernel" in n:
            kind = "conv_fwd" if "conv_igemm" in n else "wgrad"
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            s = out.setdefault(kind, [0.0, 0])
            s[0] += t
            s[1] += e.count
    return {k: {"total_us": round(v[0], 1), "launches": v[1]} for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    res = {"bench": "amp_train_step", **gpu_info(), "steps": args.steps, "modules": {}}
    for name, (mod, fwd) in cases().items():
        r = {m: [] for m in MODES}
        for m, mode in MODES.items():
            for _ in range(args.warmup):
                step(mod, fwd, mode)
        for _ in range(args.rounds):                  # alternated: every round times each mode once
            for m, mode in MODES.items():
                r[m].append(round(timed(mod, fwd, mode, args.steps), 3))
        mem = {}
        for m, mode in MODES.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            step(mod, fwd, mode)
            torch.cuda.synchronize()
            mem[m] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
        entry = {"ms": r, "speedup_fp16": round(min(r["fp32"]) / min(r["fp16"]), 3),
                 "speedup_bf16": round(min(r["fp32"]) / min(r["bf16"]), 3), "peak_mib": mem}
        if not name.startswith(("deeplab", "upsampling")):
            entry["kernels"] = {m: kernel_times(mod, fwd, mode) for m, mode in MODES.items()}
        res["modules"][name] = entry
        print(name, json.dumps(entry), file=sys.stderr)
    res.update({k: v for k, v in gpu_info().items() if k.startswith("sm_clock")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
