"""Times the eval-mode Prediction model (nuScenes Prediction.yml gates: segmentation, instance center / offset / flow;
N_FUTURE_FRAMES = 4) entering after the encoder, as bench.py enters the perception model: lift-splat -> temporal model
-> present distribution -> future prediction -> decoder on 6 cameras x 3 frames, 200 x 200 BEV.

Reported per batch (default 1 and 2):
  - the step time, eager (STP3.forward_features) and as one CUDA graph (GraphedPerception): median of --reps steps
    timed with CUDA events after --warmup steps, the two arms alternating;
  - the eager step per stage from the model's CUDA-event marks (a separate pass): temporal model, distribution, future
    prediction, decoder;
  - the same stages in torch eager fp32 (TF32 off, cuDNN) on the oracle restatements (oracle/torch_dense.py,
    oracle/torch_predict.py) on the same weights;
  - every kernel of csrc/predict_kernels.cu at the stage's 200^2 shapes: time per launch (CUDA events over --kreps
    launches) and achieved bytes/s against its byte floor (every element it must read or write once, 4 bytes per
    hi/lo element, 4 per fp32 parameter), next to the H100 SXM data sheet's 3.35 TB/s.
The card's name and power limit are read in the same run.  Prints one JSON object (and writes it to --out if given).

    python tools/predict_bench.py [--batch 1 2] [--reps 20] [--warmup 5] [--kreps 200] [--out file.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True)
    return out.stdout.strip()


def stage_flops(B, S=3, nf=4, HW=200 * 200, c=64, latent=32):
    """Multiply-adds x 2 of the prediction stage's convolutions (the per-pixel kernels are not counted)."""
    k3, k7 = 9, 49
    gru = lambda cin: 2 * HW * (k3 * cin * 2 * c + k3 * cin * c)          # [update | reset] + proposal
    dual = (S - 1) * gru(2 * c) + nf * (gru(latent + c) + gru(2 * c) + 2 * HW * k3 * c * c +
                                         2 * HW * (k7 * 2 * c * c + c * c + k3 * c * c + 2 * c * c + 2 * c))
    block = lambda n: n * 2 * HW * (k7 * c + 2 * 4 * c * c)
    spatial = 2 * ((S + nf) * (gru(2 * c) + 2 * HW * c * c))
    head = (S + nf) * 2 * HW * (128 * c + 3 * k3 * 128 * c + 4 * 128 * 128 + k3 * 128 * 128 + 128 * c)
    return B * (dual + block(nf) + block(S + nf) + spatial + head)


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kreps", type=int, default=200)
    ap.add_argument("--out", default=None)
    return ap.parse_args(argv)


def main(argv=None):
    args = parse(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("predict_bench.py measures on the GPU; no CUDA device is visible")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from oracle.make_golden_predict import build_prediction_model, predict_cfg
    from oracle import torch_dense as TD
    from oracle import torch_predict as TP
    from stp3_b200 import dense, ops
    from stp3_b200.models.stp3 import GraphedPerception
    from stp3_b200.utils import synthetic as syn

    dev = torch.device("cuda")
    res = {"gpu": gpu_info(), "workload": "nuScenes Prediction gates, 6 cameras x 3 frames, 200x200 BEV, 4 future "
           "frames, entering after the encoder", "batches": {}}
    cfg = predict_cfg(False)
    model = build_prediction_model(cfg).to(dev)
    lcfg = syn.CONFIGS["perceive"]

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    for B in args.batch:
        inp = syn.stack_samples(lcfg, list(range(B)))
        feat, depth = inp["feat"].to(dev), inp["depth_logits"].to(dev)
        host = (inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        eager = lambda: model.forward_features(feat, depth, *host)
        with torch.no_grad():
            g = GraphedPerception(model, B, lcfg.n_cameras)
            graph = lambda: g(feat, depth, *host)
            for _ in range(args.warmup):
                eager()
                graph()
            times = {"eager": [], "graph": []}
            for _ in range(args.reps):
                for name, fn in (("eager", eager), ("graph", graph)):
                    torch.cuda.synchronize()
                    a = ev()
                    fn()
                    b = ev()
                    b.synchronize()
                    times[name].append(a.elapsed_time(b))
            # stages of the eager step from the model's marks
            stage = {k: [] for k in ("temporal_model", "distribution", "future_prediction", "decoder")}
            for _ in range(args.reps):
                model.stage_events = []
                eager()
                torch.cuda.synchronize()
                m = dict(model.stage_events)
                model.stage_events = None
                stage["temporal_model"].append(m["lift_splat"].elapsed_time(m["temporal_model"]))
                stage["distribution"].append(m["start_predict"].elapsed_time(m["distribution"]))
                stage["future_prediction"].append(m["distribution"].elapsed_time(m["future_prediction"]))
                stage["decoder"].append(m["future_prediction"].elapsed_time(m["decoder"]))
            del g
            # torch eager fp32 on the oracle restatements, from the same BEV features
            prep = model.prepare_inputs(*host)
            off, r, dim = model._bev_host()
            bev = ops.lift_splat(feat, depth, *(prep[k].to(dev) for k in ("cam_M", "cam_t", "ego_R", "ego_t")),
                                 *model._axes(), off, r, dim, float(model.discount))
            S = model.receptive_field
            x = torch.cat([bev, prep["const"].to(dev).view(B, S, 6, 1, 1).expand(B, S, 6, *bev.shape[-2:])], 2)
            torch_stage = {k: [] for k in stage}
            for i in range(args.warmup + args.reps):
                e0 = ev()
                st = TD.temporal_model(x, model.temporal_model)
                e1 = ev()
                mu = TP.distribution(st[:, -1:], model.present_distribution)[:, :, :model.latent_dim]
                e2 = ev()
                xs = mu.view(B, 1, -1, 1, 1).expand(B, 1, mu.shape[-1], *st.shape[-2:])
                fut = TP.future_prediction(xs, st, model.future_prediction)
                e3 = ev()
                TD.decoder(fut, model.decoder)
                e4 = ev()
                e4.synchronize()
                if i >= args.warmup:
                    for k, (a, b) in zip(torch_stage, ((e0, e1), (e1, e2), (e2, e3), (e3, e4))):
                        torch_stage[k].append(a.elapsed_time(b))
        med = lambda v: round(statistics.median(v), 3)
        fl = stage_flops(B)
        res["batches"][B] = {
            "step_ms": {k: med(v) for k, v in times.items()},
            "step_ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
            "eager_stage_ms": {k: med(v) for k, v in stage.items()},
            "torch_fp32_stage_ms": {k: med(v) for k, v in torch_stage.items()},
            "prediction_stage_conv_flop": fl,
            "prediction_stage_tflops_achieved": round(fl / (med(stage["distribution"]) + med(stage["future_prediction"]))
                                                      / 1e9, 1),
        }
        print(json.dumps({B: res["batches"][B]}), flush=True)

    # ---------------------------------------------------------------------------------------------- kernels
    H = W = 200
    C = 64
    gen = torch.Generator(device=dev).manual_seed(0)

    def hl(T, cs):
        v = torch.randn((1, T, H, W, cs), generator=gen, device=dev)
        hi = v.to(torch.bfloat16)
        return dense.HL(hi, (v - hi.float()).to(torch.bfloat16), cs)

    buf, g128, ht, mix, t64, big = hl(1, 192), hl(1, 128), hl(1, 64), hl(1, 128), hl(1, 64), hl(1, 256)
    stack = hl(7, 64)
    gam, bet = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    gam4, bet4 = torch.ones(4 * C, device=dev), torch.zeros(4 * C, device=dev)
    w49 = torch.randn((49, C), generator=gen, device=dev) * 0.1
    w2 = torch.randn((2, C), generator=gen, device=dev) * 0.1
    vec = torch.randn((1, 64), generator=gen, device=dev)
    px, e = H * W, 4          # pixels, bytes per hi/lo element
    kernels = {
        "stp3_gru_gates": (lambda: dense.gru_gates((g128, 64), buf, (buf, 128), C), 3 * px * C * e),
        "stp3_gru_update (2 outputs)": (lambda: dense.gru_update(g128, buf, ht, buf, C, out2=(stack, 0, 3)),
                                        5 * px * C * e),
        "stp3_channel_norm_act (LN+GELU, +GELU(y))": (
            lambda: dense.channel_norm_act(t64, ht, C, ln=(gam, bet, 1e-6), gelu=True, y=t64, gelu_y=True),
            3 * px * C * e + 2 * C * 4),
        "stp3_channel_norm_act (GELU, 256 ch)": (lambda: dense.channel_norm_act(big, big, 4 * C, gelu=True),
                                                 2 * px * 4 * C * e),
        "stp3_dw_ln (7x7)": (lambda: dense.dw_ln(t64, w49, gam, 7, (gam, bet, 1e-6), ht, C),
                             2 * px * C * e + 52 * C * 4),
        "stp3_trust_mix (3 outputs)": (lambda: dense.trust_mix(t64, w2, (mix, 0), (mix, 64), [(buf, 0), (buf, 64),
                                                                                            (stack, 0, 3)], C),
                                       6 * px * C * e + 2 * C * 4),
        "stp3_maxpool2_pad (200 -> 100)": (lambda: dense.maxpool2_pad(t64), (px + px // 4) * C * e),
        "stp3_hl_copy": (lambda: dense.hl_copy((stack, 0, 0), (buf, 64), C, T=1), 2 * px * C * e),
        "stp3_hl_broadcast (32 ch)": (lambda: dense.hl_broadcast(vec, (buf, 64), 32), px * 32 * e),
    }
    kres = {}
    with torch.no_grad():
        for name, (fn, nbytes) in kernels.items():
            for _ in range(10):
                fn()
            a = ev()
            for _ in range(args.kreps):
                fn()
            b = ev()
            b.synchronize()
            us = a.elapsed_time(b) / args.kreps * 1e3
            kres[name] = {"us": round(us, 2), "byte_floor": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1),
                          "of_hbm_peak": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
            print(f"{name:44s} {us:8.2f} us  {nbytes / us / 1e3:8.1f} GB/s", flush=True)
    res["kernels_200x200"] = kres
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
