"""Cost of the deterministic mode (torch.use_deterministic_algorithms; DESIGN.md §3.14), each pair alternated in one
process, default first:
  - the lift-splat forward, default (fp32 atomics) and 64-bit fixed point, at the perceive shape (B = 4, 6 cameras x 3
    frames, 200 x 200, C = 64, pool sums, bf16 hi/lo output) and the stress shape (B = 8 per GPU, S = 5, 400 x 400,
    C = 128);
  - stp3_spatial_sum and stp3_spatial_sum_det on 12 images of 200 x 200 x 64;
  - an eager eval perceive step (encoder outputs -> lift-splat -> TemporalModel -> Decoder, B = 4) with and without the
    flag: the flag also turns off the convolution autotuner (untuned tilings);
  - full-size train steps of the TemporalModel and the Decoder (tools/amp_train_bench.py's modules, fp32).
Also reads the GPU name, power limit and SM clocks in the same run.  Prints one JSON line.

    python tools/deterministic_bench.py [--iters 20] [--rounds 3]
"""
import argparse
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import amp_train_bench as AB  # noqa: E402
import bench as BN  # noqa: E402
from stp3_b200 import dense, ops  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402

DEV = "cuda:0"


@contextlib.contextmanager
def mode(det):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def time_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def alternate(fn, iters, rounds, warmup=3):
    """{'default': [ms per round], 'deterministic': [...]}; both modes warmed up, then alternated round by round"""
    res = {"default": [], "deterministic": []}
    for det in (False, True):
        with mode(det):
            for _ in range(warmup):
                fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for det in (False, True):
            with mode(det):
                res["deterministic" if det else "default"].append(round(time_ms(fn, iters), 4))
    res["ratio"] = round(min(res["deterministic"]) / min(res["default"]), 3)
    return res


def lift_case(cfg, batch, channels_last_out):
    p = BN.make_problem(cfg, batch, 0)
    inp = p["inp"]
    feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)
    geo = (*p["mats"], *p["axes"], p["off"], p["res"], p["dim"])
    nx, ny = int(p["dim"][0]), int(p["dim"][1])
    B, S, C = feat.shape[0], feat.shape[1], feat.shape[3]
    ws = ops.Workspace()
    out_hilo = torch.empty((2, B, S, nx, ny, C), dtype=torch.bfloat16, device=DEV) if channels_last_out else None

    def run():
        ops.lift_splat(feat, depth, *geo, cfg.discount, pool_sum=True, workspace=ws, out_hilo=out_hilo)
    return run, dict(B=B, S=S, N=feat.shape[2], C=C, X=nx, Y=ny)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    res = {"bench": "deterministic_mode", **AB.gpu_info(), "iters": args.iters, "rounds": args.rounds, "ms": {}}

    for name, cfg, batch in (("lift_splat_perceive_b4", syn.CONFIGS["perceive"], 4),
                             ("lift_splat_stress_b8", syn.CONFIGS["stress"], 8)):
        run, shape = lift_case(cfg, batch, True)
        res["ms"][name] = {**alternate(run, args.iters, args.rounds), "shape": shape}
        print(name, json.dumps(res["ms"][name]), file=sys.stderr)
        del run
        torch.cuda.empty_cache()

    g = torch.Generator().manual_seed(0)
    x = torch.randn(12, 1, 200, 200, 64, generator=g)
    hl = dense.HL(x.to(torch.bfloat16).to(DEV), (x - x.to(torch.bfloat16).float()).to(torch.bfloat16).to(DEV), 64)
    res["ms"]["spatial_sum_12x200x200x64"] = alternate(lambda: dense.spatial_sum(hl), args.iters * 5, args.rounds)

    cfg = syn.CONFIGS["perceive"]
    model = BN.build_model(DEV, cfg)
    p = BN.make_problem(cfg, 4, 0)
    inp = p["inp"]
    feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)

    def perceive():
        with torch.no_grad():
            model.forward_features(feat, depth, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    res["ms"]["eval_perceive_step_b4_eager"] = alternate(perceive, max(3, args.iters // 2), args.rounds)
    del model
    torch.cuda.empty_cache()

    for name, (mod, fwd) in AB.cases().items():
        if not name.startswith(("temporal_model", "decoder")):
            continue
        res["ms"][f"train_step_{name}"] = alternate(lambda: AB.step(mod, fwd, None), max(3, args.iters // 2),
                                                    args.rounds)
        print(name, json.dumps(res["ms"][f"train_step_{name}"]), file=sys.stderr)
    res.update({k + "_after": v for k, v in AB.gpu_info().items() if k.startswith("sm_clock")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
