"""Oracle-driven precision plan for the dense path (test / analysis tool; runs on the CPU, imports oracle/).

The tensor-core convolutions carry fp32 tensors as 16-bit planes.  This script evaluates, at the HEADLINE size (one perceive
sample: 3 frames x 200x200x64 BEV, ASPP dilations 12/24/36 live), what each storage format of the activations costs
in logit error against the fp64 oracle, by re-running the oracle's own functional graph with every STORED tensor
rounded the way the kernels would store it:

    f16x2   fp16 hi + fp16 lo   (22 significand bits, ~fp32)         3 MMAs per product
    bf16x2  bf16 hi + bf16 lo   (16 bits; the round-1 format)        3 MMAs per product
    f16     ONE fp16 plane      (11 bits)                            2 MMAs (A x [W_hi; W_lo]) and half the bytes
    bf16    ONE bf16 plane      (8 bits)                             2 MMAs
weights stay hi+lo (exact to 2^-22) unless --w1 (single fp16 plane: 1 MMA per product).

    python tools/precision_plan.py [--hw 200] [--plans all-f16 ...]
Prints max |err| / max |logit| per head for every plan.
"""
import argparse
import copy
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import lift_splat_oracle as O  # noqa: E402
from oracle import torch_dense as TD  # noqa: E402
from stp3_b200.utils import geometry as G  # noqa: E402
from stp3_b200.utils import synthetic as syn  # noqa: E402


def rnd(x, fmt):
    """fp64 tensor rounded to what a stored plane set can represent."""
    if fmt == "exact":
        return x
    if fmt == "f16":
        return x.to(torch.float16).double()
    if fmt == "bf16":
        return x.float().to(torch.bfloat16).double()
    if fmt == "f16x2":
        hi = x.to(torch.float16).double()
        return hi + (x - hi).to(torch.float16).double()
    if fmt == "bf16x2":
        hi = x.float().to(torch.bfloat16).double()
        return hi + (x - hi).float().to(torch.bfloat16).double()
    raise ValueError(fmt)


class Plan:
    """storage format per stored tensor: `default`, overridden by the first matching prefix in `over`."""

    def __init__(self, default, over=(), w="exact"):
        self.default, self.over, self.w = default, list(over), w
        self.maxabs = {}

    def fmt(self, name):
        for pref, f in self.over:
            if name.startswith(pref):
                return f
        return self.default

    def __call__(self, x, name):
        m = float(x.abs().max())
        self.maxabs[name] = max(self.maxabs.get(name, 0.0), m)
        return rnd(x, self.fmt(name))

    def weight(self, w):
        return rnd(w, self.w)


def fold(conv_w, bn, q):
    """BN folded into the weights like the packed kernels do, then rounded like the weight planes."""
    s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    w = conv_w * s.view(-1, *([1] * (conv_w.dim() - 1)))
    b = bn.bias - bn.running_mean * s
    return q.weight(w), b


def cna3(x, seq, q):
    w, b = fold(seq.conv.weight, seq.norm, q)
    return F.relu(F.conv3d(x, w, b))


def causal(x, m, q):
    kt, kh, kw = m.conv.kernel_size
    x = F.pad(x, ((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0))
    w, b = fold(m.conv.weight, m.norm, q)
    return F.relu(F.conv3d(x, w, b))


def temporal_block(x, blk, q, name):
    p = blk.convolution_paths
    m0 = q(cna3(x, p[0][0], q), name + ".mid0")
    m1 = q(cna3(x, p[1][0], q), name + ".mid1")
    paths = [q(causal(m0, p[0][1], q), name + ".path0"), q(causal(m1, p[1][1], q), name + ".path1"),
             q(cna3(x, p[2], q), name + ".path2")]
    r = torch.cat(paths, 1)
    if blk.use_pyramid_pooling:
        r = torch.cat([r, TD.pyramid_pooling(x, blk.pyramid_pooling)], 1)      # enters as an fp32 bias on the device
    r = cna3(r, blk.aggregation[0], q)
    if blk.projection is not None:
        w, b = fold(blk.projection[0].weight, blk.projection[1], q)
        x = q(F.conv3d(x, w, b), name + ".res")
    return q(x + r, name + ".out")


def deeplab_head(x, head, q, name):
    aspp = head[0]
    outs = []
    for i, br in enumerate(aspp.convs):
        first = br[0]
        if isinstance(first, torch.nn.AdaptiveAvgPool2d):
            y = x.mean(dim=(2, 3), keepdim=True)
            y = F.relu(TD._bn(F.conv2d(y, br[1].weight), br[2]))
            y = y.expand(-1, -1, *x.shape[-2:])
        else:
            w, b = fold(first.weight, br[1], q)
            y = q(F.relu(F.conv2d(x, w, b, padding=first.padding, dilation=first.dilation)), f"{name}.aspp{i}")
        outs.append(y)
    w, b = fold(aspp.project[0].weight, aspp.project[1], q)
    y = q(F.relu(F.conv2d(torch.cat(outs, 1), w, b)), name + ".proj")
    w, b = fold(head[1].weight, head[2], q)
    y = q(F.relu(F.conv2d(y, w, b, padding=1)), name + ".conv3")
    return q(F.conv2d(y, q.weight(head[4].weight), head[4].bias), name + ".cls")


def temporal_model(x, tm, q):
    y = x.permute(0, 2, 1, 3, 4)
    for i, blk in enumerate(tm.model):
        y = temporal_block(y, blk, q, f"tm.block{i}")
    y = y.permute(0, 2, 1, 3, 4).contiguous()
    b, s, c, h, w = y.shape
    return deeplab_head(y.view(b * s, c, h, w), tm.final_conv, q, "tm.head").view(b, s, -1, h, w)


def basic_block(x, blk, q, name):
    w, b = fold(blk.conv1.weight, blk.bn1, q)
    y = q(F.relu(F.conv2d(x, w, b, stride=blk.conv1.stride, padding=1)), name + ".c1")
    w, b = fold(blk.conv2.weight, blk.bn2, q)
    y = F.conv2d(y, w, b, padding=1)
    if blk.downsample is not None:
        w, b = fold(blk.downsample[0].weight, blk.downsample[1], q)
        x = q(F.conv2d(x, w, b, stride=blk.downsample[0].stride), name + ".ds")
    return q(F.relu(y + x), name + ".out")


def upsampling_add(x, skip, up, q, name):
    w, b = fold(up.upsample_layer[1].weight, up.upsample_layer[2], q)
    low = q(F.conv2d(x, w, b), name + ".low")                      # the device runs the 1x1 at low resolution
    return q(F.interpolate(low, scale_factor=2, mode='bilinear', align_corners=False) + skip, name + ".out")


def head(x, h, q):
    w, b = fold(h[0].weight, h[1], q)
    y = F.relu(F.conv2d(x, w, b, padding=1))                       # stays in registers (fused 1x1 head, fp32)
    return F.conv2d(y, h[3].weight, h[3].bias)


def decoder(x, dec, q):
    b, s, c, h, w = x.shape
    x = x.reshape(b * s, c, h, w)
    skip1 = x
    wt, bs = fold(dec.first_conv.weight, dec.bn1, q)
    y = q(F.relu(F.conv2d(x, wt, bs, stride=2, padding=3)), "dec.first")
    for i, blk in enumerate(dec.layer1):
        y = basic_block(y, blk, q, f"dec.layer1.{i}")
    skip2 = y
    for i, blk in enumerate(dec.layer2):
        y = basic_block(y, blk, q, f"dec.layer2.{i}")
    skip3 = y
    for i, blk in enumerate(dec.layer3):
        y = basic_block(y, blk, q, f"dec.layer3.{i}")
    y = upsampling_add(y, skip3, dec.up3_skip, q, "dec.up3")
    y = upsampling_add(y, skip2, dec.up2_skip, q, "dec.up2")
    y = upsampling_add(y, skip1, dec.up1_skip, q, "dec.up1")
    out = {"segmentation": head(y, dec.segmentation_head, q).view(b, s, -1, h, w),
           "pedestrian": head(y, dec.pedestrian_head, q).view(b, s, -1, h, w),
           "hdmap": head(y.view(b, s, *y.shape[1:])[:, dec.n_present - 1], dec.hdmap_head, q)}
    return out


PLANS = {
    "exact (self-check)": Plan("exact"),
    "bf16x2 everywhere (round 1)": Plan("bf16x2"),
    "f16x2 everywhere": Plan("f16x2"),
    "f16 everywhere": Plan("f16"),
    "f16 everywhere, weights one fp16 plane": Plan("f16", w="f16"),
    "f16x2 storage, weights one fp16 plane": Plan("f16x2", w="f16"),
    "bf16 everywhere": Plan("bf16"),
    "f16 temporal model, f16x2 decoder": Plan("f16", [("dec.", "f16x2")]),
    "f16 DeepLab head only (rest f16x2)": Plan("f16x2", [("tm.head", "f16")]),
    "f16, BEV input f16x2": Plan("f16", [("bev", "f16x2")]),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hw", type=int, default=200, help="BEV side (200 = perceive; smaller = quick look)")
    ap.add_argument("--plans", nargs="*", default=None)
    ap.add_argument("--tilt", type=float, default=0.0)
    ap.add_argument("--sweep", action="store_true", help="one plan per stored tensor: that tensor f16, the rest f16x2")
    args = ap.parse_args()
    import bench
    cfg = syn.CONFIGS["perceive"]
    if args.hw != 200:
        half = args.hw * 0.25
        cfg = syn.LiftSplatConfig(x_bound=(-half, half, 0.5), y_bound=(-half, half, 0.5))
    torch.set_grad_enabled(False)
    model = bench.build_model(lcfg=cfg).double()
    inp = syn.lift_inputs(cfg, 1, seed=0, tilt_deg=args.tilt)
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    t0 = time.time()
    ora = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), cam_M.numpy(), cam_t.numpy(), ego_R.numpy(),
                       ego_t.numpy(), xs.numpy(), ys.numpy(), ds.numpy(), G.bev_offset(start, res).numpy(), res.numpy(),
                       dim.numpy(), cfg.discount)
    bev = torch.from_numpy(ora["bev"])
    X, Y = bev.shape[-2:]
    ego = inp["future_egomotion"].double()
    ego = torch.cat([torch.zeros_like(ego[:, :1]), ego[:, :-1]], 1)
    const = ego.view(1, -1, 6, 1, 1).expand(1, ego.shape[1], 6, X, Y)
    print(f"# perceive sample, BEV {X}x{Y}, oracle lift-splat {time.time() - t0:.0f} s, max |bev| {float(bev.abs().max()):.3g}")
    ref = None
    plans = dict(PLANS)
    if args.sweep:
        probe = Plan("exact")
        x = torch.cat([probe(bev, "bev"), const], dim=2)
        decoder(temporal_model(x, model.temporal_model, probe), model.decoder, probe)
        plans = {"exact (self-check)": Plan("exact")}
        for tname in probe.maxabs:
            plans[f"only {tname} f16"] = Plan("f16x2", [(tname, "f16")])
        args.plans = None
    for name, plan in plans.items():
        if args.plans and not any(p in name for p in args.plans) and not name.startswith("exact"):
            continue
        t0 = time.time()
        x = torch.cat([plan(bev, "bev"), const], dim=2)
        states = temporal_model(x, model.temporal_model, plan)
        out = decoder(states, model.decoder, plan)
        out["states"] = states
        if ref is None:
            ref = out
            o2 = TD.decoder(TD.temporal_model(torch.cat([bev, const], 2), model.temporal_model), model.decoder)
            chk = max(float((out[k] - o2[k]).abs().max() / o2[k].abs().max()) for k in ("segmentation", "pedestrian", "hdmap"))
            print(f"# self-check vs oracle/torch_dense.py: {chk:.1e}; largest stored magnitudes: "
                  + ", ".join(f"{k} {v:.3g}" for k, v in sorted(plan.maxabs.items(), key=lambda kv: -kv[1])[:6]))
            continue
        errs = {k: float((out[k] - ref[k]).abs().max() / ref[k].abs().max()) for k in ("states", "segmentation", "pedestrian", "hdmap")}
        print(f"{name:45s} " + "  ".join(f"{k} {v:.2e}" for k, v in errs.items()) + f"   ({time.time() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main()
