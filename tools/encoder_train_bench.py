"""Train-mode encoder heads at the Perception size (M = B*S*N = 4*3*6 = 72 images, r_lo 56 x 28 x 60, r_hi 160 x 14 x 30,
C = 64 context channels, D = 48 depth bins), timed with CUDA events after warm-up:

  (a) forward + backward of the two heads, whole and per stage: the DeepLab halves (DeepLabHead(160, 160, hidden 64),
      input requiring grad) and the UpsamplingConcat halves (216 -> 64 channels-last, 216 -> 48), both inputs
      requiring grad;
  (b) the lift-splat backward for channels-last features: stp3_lift_splat_bwd_cl against stp3_lift_splat_bwd between two
      transposing copies (features to NCHW, their gradient back), alternated in this process, `--repeats` windows each,
      median and min..max printed; the two results are compared bit for bit.

Prints one JSON line with the GPU name, power limit and SM clock read in the same run and the algorithmic flops /
bytes computed from the shapes.  Needs a GPU (there is no CPU path).

    python tools/encoder_train_bench.py [--steps 10] [--warmup 3] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stp3_b200 import ops  # noqa: E402
from stp3_b200.layers.convolutions import DeepLabHead, UpsamplingConcat  # noqa: E402
from stp3_b200.utils import geometry as G  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402
from tools.head_train_bench import gpu_info, timed  # noqa: E402

B = 4
C_LO, C_HI, HIDDEN = 56, 160, 64


def conv_flops(m, h, w, cin, cout, k):
    return 2.0 * m * h * w * cin * cout * k * k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_train_bench needs a CUDA device (there is no CPU path)")
    dev = "cuda:0"
    cfg = syn.CONFIGS["perceive"]
    S, N, C, D = cfg.receptive_field, cfg.n_cameras, cfg.out_channels, cfg.n_depth
    Hf, Wf = cfg.feat_hw
    M = B * S * N
    gen = torch.Generator().manual_seed(5)
    r_lo = syn.exact_gauss((M, C_LO, Hf, Wf), gen).to(dev).requires_grad_(True)
    r_hi = syn.exact_gauss((M, C_HI, Hf // 2, Wf // 2), gen).to(dev).requires_grad_(True)
    mods = {"feature_layer_1": DeepLabHead(C_HI, C_HI, hidden_channel=HIDDEN), "feature_layer_2": UpsamplingConcat(C_HI + C_LO, C),
            "depth_layer_1": DeepLabHead(C_HI, C_HI, hidden_channel=HIDDEN), "depth_layer_2": UpsamplingConcat(C_HI + C_LO, D)}
    for i, m in enumerate(mods.values()):
        syn.init_exact(m, seed=3 + i).to(dev).train()
    g_hi = syn.exact_gauss((M, C_HI, Hf // 2, Wf // 2), gen).to(dev) * 0.25
    g_feat = syn.exact_gauss((M, Hf, Wf, C), gen).to(dev) * 0.25
    g_depth = syn.exact_gauss((M, D, Hf, Wf), gen).to(dev) * 0.25

    def zero():
        r_lo.grad = r_hi.grad = None
        for m in mods.values():
            m.zero_grad(set_to_none=True)

    def deeplab(name):
        def step():
            zero()
            (mods[name](r_hi) * g_hi).sum().backward()
        return step

    def upcat(name, g, channels_last):
        def step():
            zero()
            (mods[name](r_hi, r_lo, channels_last=channels_last) * g).sum().backward()
        return step

    def both():
        zero()
        f = mods["feature_layer_2"](mods["feature_layer_1"](r_hi), r_lo, channels_last=True)
        d = mods["depth_layer_2"](mods["depth_layer_1"](r_hi), r_lo)
        ((f * g_feat).sum() + (d * g_depth).sum()).backward()

    res = {"heads_fwd_bwd_ms": timed(both, args.steps, args.warmup),
           "feature_deeplab_fwd_bwd_ms": timed(deeplab("feature_layer_1"), args.steps, args.warmup),
           "depth_deeplab_fwd_bwd_ms": timed(deeplab("depth_layer_1"), args.steps, args.warmup),
           "feature_upconcat_fwd_bwd_ms": timed(upcat("feature_layer_2", g_feat, True), args.steps, args.warmup),
           "depth_upconcat_fwd_bwd_ms": timed(upcat("depth_layer_2", g_depth, False), args.steps, args.warmup)}
    # forward + input gradient + weight gradient of the two 3x3 convolutions of an UpsamplingConcat
    for name, cout in (("feature", C), ("depth", D)):
        fl = 3.0 * (conv_flops(M, Hf, Wf, C_HI + C_LO, cout, 3) + conv_flops(M, Hf, Wf, cout, cout, 3))
        res[f"{name}_upconcat_conv_gflop"] = fl / 1e9
        res[f"{name}_upconcat_conv_tflops"] = fl / (res[f"{name}_upconcat_fwd_bwd_ms"] * 1e-3) / 1e12
    zero()

    # ---- (b) lift-splat backward for channels-last features
    inp = syn.lift_inputs(cfg, B, seed=3, random_pose=True)
    cam = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    axes = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    bev_res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    geo = tuple(t.to(dev) for t in cam + tuple(axes)) + (G.bev_offset(start, bev_res), bev_res, dim, cfg.discount)
    feat_cl = inp["feat"].permute(0, 1, 2, 4, 5, 3).contiguous().to(dev)
    depth = inp["depth_logits"].to(dev)
    X, Y = int(dim[0]), int(dim[1])
    g_out = syn.exact_gauss((B, S, C, X, Y), gen).to(dev)
    keep = {}

    def nchw_plus_transposes():
        gf, gd = ops.lift_splat_backward(g_out, feat_cl.permute(0, 1, 2, 5, 3, 4).contiguous(), depth, *geo)
        keep["nchw"] = (gf.permute(0, 1, 2, 4, 5, 3).contiguous(), gd)

    def channels_last():
        keep["cl"] = ops.lift_splat_backward(g_out, feat_cl, depth, *geo, feat_channels_last=True)

    t_nchw, t_cl = [], []
    for _ in range(args.repeats):
        t_nchw.append(timed(nchw_plus_transposes, args.steps, args.warmup))
        t_cl.append(timed(channels_last, args.steps, args.warmup))
    same = all(torch.equal(a, b) for a, b in zip(keep["nchw"], keep["cl"]))
    f_bytes, d_bytes, o_bytes = 4.0 * M * C * Hf * Wf, 4.0 * M * D * Hf * Wf, 4.0 * B * S * C * X * Y
    # compulsory traffic: grad_out read and the pillar-major gradient grid written and read once; features and depth
    # logits read, their gradients written (the gathers of the grid per frustum point are served from cache at best)
    min_bytes = 3 * o_bytes + 2 * f_bytes + 2 * d_bytes
    spread = lambda v: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}  # noqa: E731
    print(json.dumps({
        **gpu_info(), "M": M, "r_lo": [C_LO, Hf, Wf], "r_hi": [C_HI, Hf // 2, Wf // 2], "C": C, "D": D,
        "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
        **{k: round(v, 3) for k, v in res.items()},
        "lift_bwd_nchw_plus_transposes_ms": spread(t_nchw), "lift_bwd_channels_last_ms": spread(t_cl),
        "lift_bwd_bitwise_equal": same, "lift_bwd_min_hbm_mbytes": round(min_bytes / 1e6, 1),
        "lift_bwd_transposes_extra_mbytes": round(4 * f_bytes / 1e6, 1),
        "lift_bwd_channels_last_gbytes_per_s": round(min_bytes / (statistics.median(t_cl) * 1e-3) / 1e9, 1),
    }))


if __name__ == "__main__":
    main()
