"""Times a train step (forward + backward) of the EfficientNet-b4 trunk (cut after block 21) at 224x480: the native
train path (EfficientNetTrunk(trainable=True).train()) against torch autograd on the restatement of the same trunk
(tests/trunk_train_reference.py over oracle/efficientnet_oracle.py; cuDNN, TF32 off, channels_last) in fp32 and under
fp16 autocast.  Every arm runs with batch-statistics BatchNorm and the same pinned drop-connect masks, and the endpoints
receive the same seeded gradients.

Reported per M (default 54 = 3 samples x 3 frames x 6 cameras, and 72): the median step time of each arm (warm-up, then
--reps steps timed with CUDA events, arms alternating), max_memory_allocated per arm, the native step per stage (a
separate pass with a CUDA event around every host call; the stage of a call is the layer it serves), and the achieved
bytes/s of the depthwise backward kernels (bytes from shapes: every element read or written once) against the H100 SXM
data sheet's 3.35 TB/s.  Then one whole-model train step from camera images at --model-batch samples: model.train()
with the trainable native trunk against the frozen-trunk recipe (model.eval(); encoder.train_heads(); temporal_model
and decoder train()).  The card's name, power limit and SM clocks are read in the same run.  Prints one JSON object.

    python tools/trunk_train_bench.py [--m 54 72] [--reps 10] [--warmup 3] [--model-batch 3] [--no-model]
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
STAGE_OF = {                    # host call -> stage of the step
    "stem_raw": "stem", "stem_wgrad": "stem",
    "conv1x1_raw": "expand", "conv_raw": "projection", "conv1x1_dgrad": "projection",
    "conv_dgrad": "expand", "conv_wgrad": "1x1 and squeeze-excite weight gradients",
    "dw_raw": "depthwise", "dw_dgrad": "depthwise backward", "dw_wgrad": "depthwise backward",
    "image_channel_sums": "squeeze-excite", "se_gate": "squeeze-excite", "image_channel_dot": "squeeze-excite",
    "se_backward": "squeeze-excite", "channel_sums": "squeeze-excite",
    "bn_stats_module": "BatchNorm passes", "bn_act": "BatchNorm passes", "bn_act_grad": "BatchNorm passes",
    "bn_backward": "BatchNorm passes",
}


def dw_backward_bytes(name, args):
    """bytes the depthwise backward kernels move, from shapes (fp32, every element once)"""
    if name == "dw_dgrad":
        g, _, _, _, (H, W) = args
        return 4 * (g.numel() + g.shape[0] * H * W * g.shape[3])
    x, g = args[0], args[1]
    return 4 * (x.numel() + g.numel())


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True)
    return out.stdout.strip()


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, nargs="+", default=[54, 72])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--model-batch", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--hw", type=int, nargs=2, default=[224, 480])
    return ap.parse_args(argv)


def main(argv=None):
    args = parse(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("trunk_train_bench.py needs a CUDA device")
    from oracle import efficientnet_oracle as EO
    from stp3_b200 import dense, dense_train
    from stp3_b200.models import efficientnet as EN
    from tests import trunk_train_reference as TR

    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    H, W = args.hw
    result = {"what": "EfficientNet-b4 trunk train step (forward + backward), blocks 0-21", "image_hw": [H, W],
              "gpu": gpu_info(), "per_m": {}}

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for M in args.m:
        ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=0), 'b4')
        nat = EN.EfficientNetTrunk('b4', trainable=True)
        nat.load_state_dict(ora.state_dict(), strict=True)
        nat = nat.to(dev).train()
        ref = ora.to(dev).to(memory_format=torch.channels_last).train()
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(M, 3, H, W, device=dev, generator=gen)
        x_cl = x.contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            r3, r4 = nat.eval()(x)
        nat.train()
        g3, g4 = torch.randn(r3.shape, device=dev, generator=gen), torch.randn(r4.shape, device=dev, generator=gen)
        del r3, r4

        def native():
            torch.manual_seed(1)
            o3, o4 = nat(x)
            torch.autograd.backward([o3, o4], [g3, g4])

        def restated(amp):
            def step():
                torch.manual_seed(1)
                masks = TR.draw_masks(ref, M, dev)
                with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                    o3, o4 = TR.trunk_forward(ref, x_cl, masks)
                torch.autograd.backward([o3.float(), o4.float()], [g3, g4])
            return step

        arms = {"native": native, "torch_fp32_cudnn": restated(False), "torch_fp16_autocast": restated(True)}
        for fn in arms.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        peak = {}
        for name, fn in arms.items():
            for p in list(nat.parameters()) + list(ref.parameters()):
                p.grad = None
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            fn()
            torch.cuda.synchronize()
            peak[name] = {"max_memory_allocated_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
                          "above_inputs_gb": (torch.cuda.max_memory_allocated(dev) - base) / 1e9}
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for name, fn in arms.items():
                times[name].append(timed(fn))

        # per stage: wrap the host calls of the train path with CUDA events
        stage_ms, dw_bytes = {}, {"dw_dgrad": 0, "dw_wgrad": 0}
        dw_ms = {"dw_dgrad": 0.0, "dw_wgrad": 0.0}
        marks, depth = [], [0]
        originals = {}
        for name in STAGE_OF:
            mod = dense if name == "se_gate" else dense_train
            originals[name] = (mod, getattr(mod, name))

            def wrap(*a, _name=name, _fn=getattr(mod, name), **kw):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                depth[0] += 1
                try:
                    out = _fn(*a, **kw)
                finally:
                    depth[0] -= 1
                e1.record()
                if depth[0] == 0:             # a call made inside another (conv1x1_raw -> conv_raw) counts once
                    marks.append((_name, e0, e1, a))
                return out
            setattr(mod, name, wrap)
        try:
            per_rep = []
            for _ in range(args.reps):
                marks.clear()
                native()
                torch.cuda.synchronize()
                acc = {}
                for name, e0, e1, a in marks:
                    ms = e0.elapsed_time(e1)
                    acc[STAGE_OF[name]] = acc.get(STAGE_OF[name], 0.0) + ms
                    if name in dw_ms:
                        dw_ms[name] += ms / args.reps
                        dw_bytes[name] += dw_backward_bytes(name, a) / args.reps
                per_rep.append(acc)
            for k in per_rep[0]:
                stage_ms[k] = statistics.median(r.get(k, 0.0) for r in per_rep)
        finally:
            for name, (mod, fn) in originals.items():
                setattr(mod, name, fn)
        med = {k: statistics.median(v) for k, v in times.items()}
        result["per_m"][M] = {
            "ms_median": med, "ms_all": times, "memory": peak,
            "native_vs_torch_fp32": med["torch_fp32_cudnn"] / med["native"],
            "native_vs_torch_fp16": med["torch_fp16_autocast"] / med["native"],
            "native_stage_ms (with an event pair around every call)": stage_ms,
            "depthwise_backward": {k: {"ms": dw_ms[k], "gbytes": dw_bytes[k] / 1e9,
                                       "tb_per_s": dw_bytes[k] / (dw_ms[k] * 1e-3) / 1e12,
                                       "frac_of_3.35_tb_per_s": dw_bytes[k] / (dw_ms[k] * 1e-3) / HBM_BYTES_PER_S}
                                   for k in dw_ms},
            "tape_bytes_formula_gb": M * EN.trunk_tape_bytes('b4', H, W) / 1e9,
        }
        marks.clear()                         # the marks hold the last pass's operands
        del nat, ref, x, x_cl, g3, g4, arms, native
        torch.cuda.empty_cache()

    if not args.no_model:
        result["model_step"] = model_step(args, dev, timed)
    result["gpu_after"] = gpu_info()
    print(json.dumps(result, indent=1, default=str))


def model_step(args, dev, timed):
    """One whole-model train step from camera images: model.train() with the trainable trunk against the frozen-trunk
    recipe, same weights and inputs."""
    import torch
    import bench
    from oracle import efficientnet_oracle as EO
    from stp3_b200.models.efficientnet import EfficientNetTrunk
    from stp3_b200.models.encoder import Encoder
    from stp3_b200.utils import synthetic as syn
    B, S, N = args.model_batch, 3, 6
    H, W = args.hw
    model = bench.build_model(None)
    enc = model.encoder
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=0), 'b4')
    model.encoder = Encoder(model.cfg.MODEL.ENCODER, model.depth_channels,
                            backbone=EfficientNetTrunk('b4', trainable=True))
    model.encoder.load_state_dict({**{f"backbone.{k}": v for k, v in ora.state_dict().items()},
                                   **{k: v for k, v in enc.state_dict().items() if not k.startswith("backbone.")}},
                                  strict=True)
    model = model.to(dev)
    inp = syn.lift_inputs(syn.CONFIGS["perceive"], B, seed=0, random_pose=False)
    image = torch.randn(B, S, N, 3, H, W, device=dev)

    def step():
        out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        loss = sum(out[k].float().square().mean() for k in ("segmentation", "pedestrian", "hdmap"))
        loss.backward()

    def whole():
        model.train()

    def frozen():
        model.eval()
        model.encoder.train_heads()
        model.temporal_model.train()
        model.decoder.train()

    res = {"batch": B, "images": B * S * N}
    for name, setup in (("model.train() with the trainable trunk", whole), ("frozen trunk, train_heads()", frozen)):
        setup()
        for _ in range(args.warmup):
            model.zero_grad(set_to_none=True)
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        ms = []
        for _ in range(args.reps):
            model.zero_grad(set_to_none=True)
            ms.append(timed(step))
        res[name] = {"ms_median": statistics.median(ms), "ms_all": ms,
                     "max_memory_allocated_gb": torch.cuda.max_memory_allocated(dev) / 1e9}
    return res


if __name__ == "__main__":
    main()
