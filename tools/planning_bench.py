"""Times the eval-mode Planning head (model.planning, as evaluate.py and carla_agent.py call it) at the nuScenes and
CARLA Planning.yml sizes: N 1800 candidates, 6 frames, G 256, cam_front 64 x 28 x 60; N 2400, 4 frames, G 128,
64 x 32 x 32; both on 200 x 200 BEV maps, for B = 1 and 4.  Each call is timed with CUDA events around the whole
Python call (command windows, channel reduction, the three planning kernels), median of --reps after --warmup calls.
When the unmodified reference is installed under oracle/_ref/, its Planning runs on the same GPU, weights and inputs
(oracle/make_golden_planning.py supplies skimage's polygon rasteriser) and is timed the same way.  The card's name and
power limit are read in the same run.  Prints one JSON line.

    python tools/planning_bench.py [--batch 1 4] [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden_planning import planning_cfg, planning_module  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def inputs(carla, B, dev, seed=0):
    N, T, hf, wf = (2400, 4, 32, 32) if carla else (1800, 6, 28, 60)
    g = torch.Generator().manual_seed(seed)
    fwd = torch.randint(0, 257, (B, N, T), generator=g).float() / 64.0
    lat = torch.randint(-64, 65, (B, N, T), generator=g).float() / 64.0
    x = dict(cam_front=syn.exact_gauss((B, 64, hf, wf), g).clamp(min=0),
             trajs=torch.stack([lat.cumsum(-1), fwd.cumsum(-1), torch.zeros(B, N, T)], -1),
             gt_trajs=None, cost_volume=syn.exact_gauss((B, T, 200, 200), g) * 256.0,
             semantic_pred=torch.randint(0, 8, (B, T, 200, 200), generator=g) == 0,
             hd_map=syn.exact_gauss((B, 4, 200, 200), g) * 2.0,
             commands=(['LEFT', 'FORWARD', 'RIGHT', 'STOP'] * B)[:B],
             target_points=torch.randint(-256, 257, (B, 2), generator=g).float() / 16.0 if carla else torch.zeros(B, 2))
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in x.items()}


def time_calls(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    from oracle.ref_loader import reference_available
    ref_ok = reference_available()
    res = {"gpu": gpu_info(), "reference_installed": ref_ok, "runs": []}
    for name, carla in (("nuscenes", False), ("carla", True)):
        m = planning_module(carla).to(dev)
        ref = None
        if ref_ok:
            from oracle.make_golden_planning import load_ref_planning
            cfg = planning_cfg(carla)
            ref = load_ref_planning().Planning(cfg, 64, 6, gru_state_size=cfg.PLANNING.GRU_STATE_SIZE)
            ref.load_state_dict(m.state_dict(), strict=True)
            ref = ref.to(dev).eval()
        for B in a.batch:
            x = inputs(carla, B, dev)
            with torch.no_grad():
                row = {"config": name, "B": B, "ms": round(time_calls(lambda: m(**x), a.reps, a.warmup), 4)}
                if ref is not None:
                    row["reference_ms"] = round(time_calls(lambda: ref(**x), max(3, a.reps // 4), 1), 3)
                    _, o_ref = ref(**x)
                    _, o = m(**x)
                    row["max_abs_diff_vs_reference"] = float((o - o_ref).abs().max())
            res["runs"].append(row)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
