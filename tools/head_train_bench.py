"""Forward + backward time of the temporal model's DeepLab head in train mode (DeepLabHead(64, 64, hidden 128) on
B=2 x S=3 BEV frames of 64 x 200 x 200, input not requiring grad, as behind frozen TemporalBlocks), and of the fine-tune
step head + BEV decoder (perceive heads): the native sm_90a path against the same step in torch eager through the
train-mode restatements (oracle/torch_deeplab_train.py, oracle/torch_dense_train.py) on the same GPU, fp32 with TF32 off and fp16 autocast.  Prints one
JSON line with the GPU name, power limit and SM clock read in the same run, and the parity of the native head step
against fp64 autograd (ReLU branches and the dropout mask pinned to the native forward's).

    python tools/head_train_bench.py [--steps 10] [--warmup 3] [--hw 200 200]
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
from oracle import torch_dense_train as TT  # noqa: E402
from oracle import torch_deeplab_train as TH  # noqa: E402
from stp3_b200.layers.convolutions import DeepLabHead  # noqa: E402
from stp3_b200.models.decoder import Decoder  # noqa: E402

GATES = dict(perceive_hdmap=True, predict_pedestrian=True, predict_instance=False, predict_future_flow=False,
             planning=False)


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        p, sm, sm_max = (float(v) for v in r.stdout.strip().splitlines()[0].split(","))
        info.update(power_limit_w=p, sm_clock_mhz=sm, sm_clock_max_mhz=sm_max)
    except Exception:                               # noqa: BLE001  (reported as unknown)
        info.update(power_limit_w=None, sm_clock_mhz=None, sm_clock_max_mhz=None)
    return info


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--hw", type=int, nargs=2, default=(200, 200))
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    H, W = args.hw
    B, S = 2, 3
    head_cpu = TD.init_exact(DeepLabHead(64, 64, hidden_channel=128), seed=3).train()
    dec_cpu = TD.init_exact(Decoder(64, 2, 3, 2, GATES), seed=2).train()
    x = TD.exact_gauss((B * S, 64, H, W), torch.Generator().manual_seed(5)).to(dev)
    G = (TD.exact_gauss((B * S, 64, H, W), torch.Generator().manual_seed(9)) * 0.25).to(dev)
    shapes = {"segmentation": (B, S, 2, H, W), "pedestrian": (B, S, 2, H, W), "hdmap": (B, 4, H, W)}
    Gd = {k: v.to(dev) for k, v in TT.upstream_grads({k: torch.empty(s) for k, s in shapes.items()}, 9).items()}

    def head_step(head, fn, autocast=False):
        def step():
            head.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                loss = (fn(head, x).float() * G).sum()
            loss.backward()
        return step

    def finetune_step(head, dec, fn_head, fn_dec, autocast=False):
        def step():
            head.zero_grad(set_to_none=True)
            dec.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                y = fn_head(head, x)
                out = fn_dec(dec, y.view(B, S, *y.shape[1:]))
                loss = sum((out[k].float() * Gd[k]).sum() for k in Gd)
            loss.backward()
        return step

    native = lambda m, t: m(t)                          # noqa: E731
    eager_head = lambda m, t: TH.deeplab_head_train(t, m)  # noqa: E731
    eager_dec = lambda m, t: TT.decoder_train(t, m)      # noqa: E731
    res = {}
    head, dec = copy.deepcopy(head_cpu).to(dev), copy.deepcopy(dec_cpu).to(dev)
    res["head_native_ms"] = timed(head_step(head, native), args.steps, args.warmup)
    res["finetune_native_ms"] = timed(finetune_step(head, dec, native, native), args.steps, args.warmup)
    del head, dec
    head, dec = copy.deepcopy(head_cpu).to(dev), copy.deepcopy(dec_cpu).to(dev)
    res["head_eager_fp32_ms"] = timed(head_step(head, eager_head), args.steps, args.warmup)
    res["head_eager_fp16_autocast_ms"] = timed(head_step(head, eager_head, True), args.steps, args.warmup)
    res["finetune_eager_fp32_ms"] = timed(finetune_step(head, dec, eager_head, eager_dec), args.steps, args.warmup)
    res["finetune_eager_fp16_autocast_ms"] = timed(finetune_step(head, dec, eager_head, eager_dec, True), args.steps,
                                                   args.warmup)
    del head, dec
    torch.cuda.empty_cache()

    # parity of one native head step against fp64 autograd, ReLU branches and dropout mask pinned to the native forward
    probe = copy.deepcopy(head_cpu).to(dev)
    torch.manual_seed(0)
    with torch.no_grad():
        _, tape = probe._train_forward(x)
    h = probe.hidden
    nchw = lambda t: (t > 0).permute(0, 3, 1, 2).double()   # noqa: E731
    queue = [nchw(tape["cat"][..., i * h:(i + 1) * h]) for i in range(len(tape["branches"]))]
    queue += [nchw(tape["v"]), nchw(tape["z"]), nchw(tape["y3"])]
    keep = (tape["z"] != 0).permute(0, 3, 1, 2)
    del tape, probe
    ref = copy.deepcopy(head_cpu).double().to(dev)
    out_ref = TH.deeplab_head_train(x.double(), ref, relu=lambda t: t * queue.pop(0), dropout_mask=keep)
    (out_ref * G.double()).sum().backward()
    del keep, queue
    head = copy.deepcopy(head_cpu).to(dev)
    torch.manual_seed(0)
    out = head(x)
    (out * G).sum().backward()
    rel = lambda a, b: ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()  # noqa: E731
    parity_out = rel(out.detach(), out_ref.detach())
    parity_grad = max(rel(p.grad, r.grad) for p, r in zip(head.parameters(), ref.parameters()))
    print(json.dumps({
        **gpu_info(), "shape": [B, S, 64, H, W], "head": "DeepLabHead(64, 64, hidden 128)", "decoder": "perceive",
        "steps": args.steps, "warmup": args.warmup, **{k: round(v, 3) for k, v in res.items()},
        "head_speedup_vs_fp32": round(res["head_eager_fp32_ms"] / res["head_native_ms"], 3),
        "head_speedup_vs_fp16": round(res["head_eager_fp16_autocast_ms"] / res["head_native_ms"], 3),
        "finetune_speedup_vs_fp32": round(res["finetune_eager_fp32_ms"] / res["finetune_native_ms"], 3),
        "finetune_speedup_vs_fp16": round(res["finetune_eager_fp16_autocast_ms"] / res["finetune_native_ms"], 3),
        "parity_logits_rel_max": parity_out, "parity_grad_rel_max": parity_grad,
    }))


if __name__ == "__main__":
    main()
