"""Forward + backward time of TemporalModel in train mode (its two TemporalBlocks and the DeepLab head; 64 BEV channels +
6 ego-motion channels, B=2 x S=3 frames of 200 x 200, input requiring grad), and of the train step lift-splat +
temporal model + BEV decoder (perceive configuration, feat / depth logits requiring grad): the native sm_90a path
against the same work in torch eager through the train-mode restatements (oracle/torch_temporal_train.py,
oracle/torch_dense_train.py) on the same GPU, fp32 with TF32 off and fp16 autocast.  The lift-splat has no torch-eager
form in this package, so the step's eager arms run it natively too (ops.lift_splat_autograd) and differ from the
native arm only after it.  Prints one JSON line with the GPU name, power limit and SM clock read in the same run, and
the parity of the native temporal-model step against fp64 autograd (ReLU branches and the dropout mask pinned to the
native forward's).

    python tools/temporal_train_bench.py [--steps 10] [--warmup 3]
"""
import argparse
import copy
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import torch_dense as TD  # noqa: E402
from oracle import torch_dense_train as TT  # noqa: E402
from oracle import torch_temporal_train as OT  # noqa: E402
from stp3_b200.models.temporal_model import TemporalModel  # noqa: E402
from tools.head_train_bench import gpu_info, timed  # noqa: E402


def full_input(x, const):
    """x (B, S, C, H, W) with the constant channels (B*S, n) broadcast behind it: the reference model's input."""
    B, S, _, H, W = x.shape
    return torch.cat([x, const.view(B, S, -1, 1, 1).expand(B, S, const.shape[1], H, W)], 2)


def perceive_stp3(dev):
    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    from stp3_b200.utils import geometry as G
    cfg = get_cfg()
    model = STP3(cfg, backbone=torch.nn.Identity())
    with torch.no_grad():
        TD.init_exact(model, seed=7)
        model.frustum.copy_(model.create_frustum())
        res, start, dim = G.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
    model = model.to(dev).train()
    model.encoder.eval()
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    B, S, H, W = 2, 3, 200, 200
    tm_cpu = TD.init_exact(TemporalModel(70, S, (H, W), start_out_channels=64), seed=3)
    tm_cpu.model[0].n_const = 6
    tm_cpu.train()
    x = TD.exact_gauss((B, S, 64, H, W), torch.Generator().manual_seed(5)).to(dev).requires_grad_(True)
    const = TD.exact_gauss((B * S, 6), torch.Generator().manual_seed(6)).to(dev)
    G = (TD.exact_gauss((B, S, 64, H, W), torch.Generator().manual_seed(9)) * 0.25).to(dev)
    res = {}

    def tm_step(tm, native, autocast=False):
        def step():
            tm.zero_grad(set_to_none=True)
            x.grad = None
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                y = tm(x, const=const) if native else OT.temporal_model_train(full_input(x, const), tm)
                loss = (y.float() * G).sum()
            loss.backward()
        return step

    tm = copy.deepcopy(tm_cpu).to(dev)
    res["temporal_native_ms"] = timed(tm_step(tm, True), args.steps, args.warmup)
    res["temporal_eager_fp32_ms"] = timed(tm_step(tm, False), args.steps, args.warmup)
    res["temporal_eager_fp16_autocast_ms"] = timed(tm_step(tm, False, True), args.steps, args.warmup)
    del tm
    torch.cuda.empty_cache()

    # the train step from the encoder's outputs: lift-splat (autograd) -> temporal model -> decoder
    from stp3_b200.utils import synthetic as syn
    inp = syn.lift_inputs(syn.LiftSplatConfig(), B, seed=4)
    feat = inp["feat"].to(dev).requires_grad_(True)
    depth = inp["depth_logits"].to(dev).requires_grad_(True)
    model = perceive_stp3(dev)
    with torch.no_grad():
        torch.manual_seed(0)
        shapes = {k: v.shape for k, v in model.forward_features(feat.detach(), depth.detach(), inp["intrinsics"],
                                                                inp["extrinsics"], inp["future_egomotion"]).items()
                  if torch.is_tensor(v) and k != "depth_prediction"}
    Gd = {k: v.to(dev) for k, v in TT.upstream_grads({k: torch.empty(s) for k, s in shapes.items()}, 9).items()}
    c = model.prepare_inputs(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])["const"].to(dev)

    def full_step(native, autocast=False):
        def step():
            model.zero_grad(set_to_none=True)
            feat.grad, depth.grad = None, None
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                if native:
                    out = model.forward_features(feat, depth, inp["intrinsics"], inp["extrinsics"],
                                                 inp["future_egomotion"])
                else:
                    bev = model.projection_to_birds_eye_view(feat, depth, inp["intrinsics"], inp["extrinsics"],
                                                             inp["future_egomotion"])
                    y = OT.temporal_model_train(full_input(bev, c), model.temporal_model)
                    out = TT.decoder_train(y, model.decoder)
                loss = sum((out[k].float() * Gd[k]).sum() for k in Gd)
            loss.backward()
        return step
    res["step_native_ms"] = timed(full_step(True), args.steps, args.warmup)
    res["step_eager_fp32_ms"] = timed(full_step(False), args.steps, args.warmup)
    res["step_eager_fp16_autocast_ms"] = timed(full_step(False, True), args.steps, args.warmup)
    del model, feat, depth
    torch.cuda.empty_cache()

    # parity of one native temporal-model step against fp64 autograd, ReLU branches and dropout mask pinned
    from tests.test_temporal_train_gpu import native_masks, oracle_step, rel_max
    xc, cc, Gc = x.detach().cpu(), const.cpu(), G.cpu()
    masks, keep = native_masks(tm_cpu, xc, cc, seed=17)
    out_ref, ref, gx_ref = oracle_step(tm_cpu, xc, cc, Gc, masks, keep)
    del masks, keep
    tm = copy.deepcopy(tm_cpu).to(dev)
    xg = x.detach().clone().requires_grad_(True)
    torch.manual_seed(17)
    out = tm(xg, const=const)
    (out * G).sum().backward()
    parity_out = rel_max(out.detach(), out_ref.detach())
    parity_grad = max([rel_max(p.grad, r.grad) for p, r in zip(tm.parameters(), ref.parameters())] +
                      [rel_max(xg.grad, gx_ref)])
    print(json.dumps({
        **gpu_info(), "shape": [B, S, 64, H, W], "n_const": 6, "temporal_model": "TemporalModel(70, 3) + DeepLabHead",
        "decoder": "perceive", "steps": args.steps, "warmup": args.warmup, **{k: round(v, 3) for k, v in res.items()},
        "temporal_speedup_vs_fp32": round(res["temporal_eager_fp32_ms"] / res["temporal_native_ms"], 3),
        "temporal_speedup_vs_fp16": round(res["temporal_eager_fp16_autocast_ms"] / res["temporal_native_ms"], 3),
        "step_speedup_vs_fp32": round(res["step_eager_fp32_ms"] / res["step_native_ms"], 3),
        "step_speedup_vs_fp16": round(res["step_eager_fp16_autocast_ms"] / res["step_native_ms"], 3),
        "parity_logits_rel_max": parity_out, "parity_grad_rel_max": parity_grad,
    }))


if __name__ == "__main__":
    main()
