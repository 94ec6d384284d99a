"""GPU: the DeepLab head in train mode (batch statistics, ASPP pooling branch over the batch, dropout, autograd) on the
sm_90a kernels.

Kernel level: dilated weight / input gradients against fp64 torch.nn.grad (taps whose window lies in the padding give
exact zeros), undilated ones bitwise equal to the values recorded before dilation existed, the dropout keep bits of
stp3_bn_apply and the per-image channel sums.  Module level: logits, running statistics and every gradient against
fp64 autograd through the train-mode restatement (oracle/torch_deeplab_train.deeplab_head_train) with the ReLU branches
and the dropout mask pinned to the native forward, determinism, a train step followed by an eval forward, the refusals.
Model level: the recipe model.eval(); final_conv.train(); decoder.train()."""
import copy
import hashlib
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import torch_dense as TD
from oracle import torch_dense_train as TT
from oracle import torch_deeplab_train as TH
from stp3_b200 import _lib, dense_train as T
from stp3_b200.layers.convolutions import DeepLabHead
from tests import train_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rel_max(got, ref):
    got, ref = got.double(), ref.double().to(got.device)
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ kernel level
DILATED = [(64, 128, d, hw) for d in (12, 24, 36) for hw in ((200, 200), (48, 64))] + \
          [(160, 64, d, (14, 30)) for d in (12, 24, 36)]


@pytest.mark.parametrize("cin,cout,d,hw", DILATED)
def test_dilated_wgrad_dgrad(cin, cout, d, hw):
    H, W = hw
    N = 2
    x = gauss((N, cin, H, W), 1).double().to(DEV)
    w = (gauss((cout, cin, 3, 3), 2).double() * 0.05).to(DEV)
    g = gauss((N, cout, H, W), 3).double().to(DEV)
    dw_ref = torch.nn.grad.conv2d_weight(x, w.shape, g, padding=d, dilation=d)
    dx_ref = torch.nn.grad.conv2d_input(x.shape, w, g, padding=d, dilation=d)
    x_cl = x.float().permute(0, 2, 3, 1).contiguous()
    g_cl = g.float().permute(0, 2, 3, 1).contiguous()
    dw = T.conv_wgrad(x_cl, g_cl, 3, 3, 1, dilation=d)
    dx = T.conv_dgrad(g_cl, w.float(), 1, H, W, dilation=d)
    torch.cuda.synchronize()
    e_w, e_x = rel_max(dw, dw_ref), rel_max(dx.permute(0, 3, 1, 2), dx_ref)
    print(f"3x3 d{d} {cin}->{cout} {H}x{W}: wgrad {e_w:.2e}, dgrad {e_x:.2e} of max")
    assert e_w < 1e-3 and e_x < 1e-3, (e_w, e_x)
    for ky in range(3):
        for kx in range(3):
            if abs((ky - 1) * d) >= H or abs((kx - 1) * d) >= W:      # the tap reads only zero padding
                assert not dw[:, :, ky, kx].any(), (ky, kx)


# sha256 of the fp32 bytes of conv_wgrad / conv_dgrad on the decoder geometries (tests/test_decoder_train_gpu.py GEOMS)
# at 48x64.  The input gradients' bits are those recorded before the dilation argument existed.  The weight gradients'
# are those of the kernel that adds each 64-pixel stage into its split's sum in fp32 (DESIGN.md 3.10); that change
# moved every split of more than one stage, and the test also holds these bits to the exact fp64 product.
UNDILATED_SHA = {
    (64, 64, 7, 2): ('6a2fa62a450633ad', '4b5adef187ff5304'),
    (64, 64, 3, 1): ('2aa21be489434ab4', '430f95c89e558827'),
    (64, 128, 3, 2): ('9fafc5c3b6d5ea19', '5fc2cd242d6b3981'),
    (128, 128, 3, 1): ('a8f88b3877946e20', '1789c9e351357897'),
    (64, 128, 1, 2): ('aef67d5228d565a4', '8f0983a4372e3699'),
    (256, 128, 1, 1): ('67c9bc8e349c2db3', 'e97b3182d03c162d'),
    (64, 1, 1, 1): ('1d0157fb760f27f8', 'a1c08de8e5c09b73'),
    (64, 8, 1, 1): ('052def36b07c8d80', '1ddbe4ef444b880a'),
}
GEOMS = [(64, 64, 7, 2), (64, 64, 3, 1), (64, 128, 3, 2), (128, 128, 3, 1), (64, 128, 1, 2), (256, 128, 1, 1),
         (64, 1, 1, 1), (64, 8, 1, 1)]


def undilated_outputs(cin, cout, k, stride):
    H, W, N = 48, 64, 2
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    x_cl = gauss((N, H, W, cin), 1).to(DEV)
    g_cl = gauss((N, Ho, Wo, cout), 3).to(DEV)
    w = (gauss((cout, cin, k, k), 2) * 0.05).to(DEV)
    return T.conv_wgrad(x_cl, g_cl, k, k, stride), T.conv_dgrad(g_cl, w, stride, H, W)


def sha(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()[:16]


@pytest.mark.parametrize("cin,cout,k,stride", GEOMS)
def test_undilated_gradients_match_recorded_bits(cin, cout, k, stride):
    dw, dx = undilated_outputs(cin, cout, k, stride)
    assert (sha(dw), sha(dx)) == UNDILATED_SHA[(cin, cout, k, stride)]
    H, W, N = 48, 64, 2
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    ref = R.wgrad(gauss((N, H, W, cin), 1).to(DEV), gauss((N, Ho, Wo, cout), 3).to(DEV), k, k, stride, (k - 1) // 2)
    assert rel_max(dw, ref[:, :, 0]) < 3e-5


def bn_apply_raw(x, p, seed, offset, n_pix=None, x_off=0):
    """stp3_bn_apply with identity statistics (mean 0, invstd 1, gamma 1, beta 0) and ReLU on rows
    [x_off, x_off + n_pix) of x (n, C) -> y of those rows."""
    n, C = x.shape
    n_pix = n if n_pix is None else n_pix
    zeros, ones = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    y = torch.empty((n_pix, C), device=DEV)
    code = _lib.lib().stp3_bn_apply(x[x_off:].data_ptr(), n_pix, C, C, zeros.data_ptr(), ones.data_ptr(),
                                    ones.data_ptr(), zeros.data_ptr(), None, 0, 1, p, seed, offset, y.data_ptr(), C,
                                    None, None, 0, torch.cuda.current_stream().cuda_stream)
    _lib.check(code, "stp3_bn_apply")
    return y


@pytest.mark.parametrize("p", [0.5, 0.1, 0.9])
def test_dropout_keep_fraction_seed_and_split(p):
    x = gauss((6 * 48 * 64, 128), 4).to(DEV)
    y = bn_apply_raw(x, p, 1234, 0)
    pos = x > 0
    n = int(pos.sum())
    kept = int((y > 0).sum())
    sigma = math.sqrt(p * (1 - p) / n)
    print(f"p {p}: kept {kept / n:.5f} of {n} positive elements (expected {1 - p}, sigma {sigma:.1e})")
    assert abs(kept / n - (1 - p)) < 6 * sigma
    assert not (y[~pos] != 0).any()
    scale = 1.0 / (1.0 - torch.tensor(p, dtype=torch.float32))              # the kernel's fp32 1 / (1 - p)
    assert torch.equal(y[y > 0], x[y > 0] * scale.to(DEV))
    assert torch.equal(y, bn_apply_raw(x, p, 1234, 0))
    assert not torch.equal(y > 0, bn_apply_raw(x, p, 1235, 0) > 0)
    # the mask is a function of (seed, offset + flat index): split at an odd row, three launches, same result
    C = x.shape[1]
    a, b = 1001, 3333
    parts = [bn_apply_raw(x, p, 1234, 0, n_pix=a), bn_apply_raw(x, p, 1234, a * C, n_pix=b, x_off=a),
             bn_apply_raw(x, p, 1234, (a + b) * C, n_pix=x.shape[0] - a - b, x_off=a + b)]
    assert torch.equal(torch.cat(parts), y)
    assert torch.equal(bn_apply_raw(x, 0.0, 1234, 0), x.clamp_min(0))


def test_image_channel_sums():
    x = gauss((6, 200, 200, 128), 5).to(DEV)
    x[..., 7] += 1000.0
    s = T.image_channel_sums(x)
    ref = x.double().sum(dim=(1, 2))
    e = ((s.double() - ref).abs() / ref.abs().clamp_min(1.0)).max().item()
    assert e < 1e-6, e
    assert torch.equal(s, T.image_channel_sums(x))


# ------------------------------------------------------------------------------------------------ module level
CONFIGS = {"temporal_48x64": (64, 64, 128, 6, 48, 64), "temporal_200x200": (64, 64, 128, 6, 200, 200),
           "encoder_14x30": (160, 160, 64, 18, 14, 30)}


def make_head(cin, ncls, hidden, momentum=0.05):
    head = TD.init_exact(DeepLabHead(cin, ncls, hidden_channel=hidden), seed=3)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = momentum
    return head.train()


def native_masks(head_cpu, x, seed):
    """(ReLU masks in the restatement's call order, dropout keep mask) of the native forward, NCHW fp64."""
    head = copy.deepcopy(head_cpu).to(DEV)
    torch.manual_seed(seed)
    with torch.no_grad():
        _, tape = head._train_forward(x.to(DEV))
    h = head.hidden
    nchw = lambda t: (t > 0).permute(0, 3, 1, 2).double()       # noqa: E731
    masks = [nchw(tape["cat"][..., i * h:(i + 1) * h]) for i in range(len(tape["branches"]))]
    masks += [nchw(tape["v"]), nchw(tape["z"]), nchw(tape["y3"])]
    return masks, tape["z"] != 0


def oracle_step(head_cpu, x, G, masks, keep):
    ref = copy.deepcopy(head_cpu).double().to(DEV)
    xd = x.double().to(DEV).requires_grad_(True)
    queue = list(masks)
    out = TH.deeplab_head_train(xd, ref, relu=lambda t: t * queue.pop(0), dropout_mask=keep.permute(0, 3, 1, 2))
    assert not queue
    (out * G.double().to(DEV)).sum().backward()
    return out, ref, xd.grad


def native_step(head, x, G, seed):
    x = x.to(DEV).requires_grad_(True)
    head.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    out = head(x)
    (out * G.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    return out, x.grad


@pytest.mark.parametrize("name", list(CONFIGS))
def test_train_step_matches_fp64_oracle(name):
    cin, ncls, hidden, N, H, W = CONFIGS[name]
    head_cpu = make_head(cin, ncls, hidden)
    x = gauss((N, cin, H, W), 5)
    G = gauss((N, ncls, H, W), 9) * 0.25
    masks, keep = native_masks(head_cpu, x, seed=17)
    out_ref, ref, gx_ref = oracle_step(head_cpu, x, G, masks, keep)
    head = copy.deepcopy(head_cpu).to(DEV)
    out, gx = native_step(head, x, G, seed=17)
    assert out.grad_fn is not None
    worst = {"out": rel_max(out.detach(), out_ref.detach())}
    for (k, b), (_, b_ref) in zip(head.named_buffers(), ref.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(b_ref) == 1, k
            continue
        e = rel_max(b, b_ref)
        assert e < 1e-5, (k, e)
    for (k, p), (_, p_ref) in zip(head.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, f"{k}: no gradient"
        worst[f"grad.{k}"] = rel_max(p.grad, p_ref.grad)
    worst["grad.x"] = rel_max(gx, gx_ref)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"{name}: {keep.float().mean().item():.3f} of the projection output kept and positive; worst {[(k, f'{v:.2e}') for k, v in top]}")
    assert worst.pop("out") < 1e-3
    bad = {k: v for k, v in worst.items() if v > 2.5e-4}
    assert not bad, bad
    if name == "temporal_200x200":             # determinism: the same seed gives the same forward and backward
        grads1 = [p.grad.clone() for p in head.parameters()] + [gx.clone()]
        out2, gx2 = native_step(head, x, G, seed=17)
        assert torch.equal(out, out2)
        assert all(torch.equal(a, b) for a, b in zip(grads1, [p.grad for p in head.parameters()] + [gx2]))


def test_dropout_seed_reproduces_forward():
    head = make_head(64, 64, 128).to(DEV)
    x = gauss((6, 64, 48, 64), 5).to(DEV)
    outs = []
    for seed in (1, 1, 2):
        torch.manual_seed(seed)
        with torch.no_grad():
            outs.append(head(x))
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0], outs[2])


def test_sgd_step_then_eval_matches_eval_oracle():
    head = make_head(64, 64, 128, 0.1).to(DEV)
    x = gauss((6, 64, 48, 64), 5).to(DEV)
    head.eval()
    with torch.no_grad():
        head(x)                                   # packs (and caches) the eval-mode weights
    head.train()
    opt = torch.optim.SGD(head.parameters(), lr=0.05)
    (head(x) ** 2).mean().backward()
    opt.step()
    head.eval()
    with torch.no_grad():
        got = head(x)
        ref = TD.deeplab_head(x.double().cpu(), copy.deepcopy(head).cpu().double())
    e = rel_max(got, ref)
    assert e < 1e-3, e


def test_no_grad_train_forward_updates_running_stats():
    head_cpu = make_head(160, 160, 64, 0.1)
    x = gauss((18, 160, 14, 30), 5)
    ref = copy.deepcopy(head_cpu).double()
    params = [p.detach().clone() for p in head_cpu.parameters()]
    _, keep = native_masks(head_cpu, x, seed=4)
    with torch.no_grad():
        TH.deeplab_head_train(x.double(), ref, dropout_mask=keep.permute(0, 3, 1, 2).cpu())
        head = copy.deepcopy(head_cpu).to(DEV)
        torch.manual_seed(4)
        out = head(x.to(DEV))
    assert out.grad_fn is None
    for (k, b), (_, b_ref) in zip(head.named_buffers(), ref.named_buffers()):
        assert rel_max(b, b_ref) < 1e-5, k
    assert all(torch.equal(p.cpu(), q) for p, q in zip(head.parameters(), params))


@pytest.mark.parametrize("what", ["n1", "sync", "momentum_none"])
def test_refusals(what):
    head = make_head(64, 64, 128)
    x = gauss((6, 64, 48, 64), 5)
    if what == "n1":
        x, exc, match = x[:1], ValueError, "Expected more than 1 value per channel"
    elif what == "sync":
        head = torch.nn.SyncBatchNorm.convert_sync_batchnorm(head)
        exc, match = NotImplementedError, "SyncBatchNorm"
    else:
        head[0].convs[4][2].momentum = None
        exc, match = NotImplementedError, "momentum=None"
    head = head.to(DEV).train()
    with pytest.raises(exc, match=match):
        head(x.to(DEV))


def test_autograd_node_guards():
    head = make_head(64, 64, 128).to(DEV)
    x = gauss((6, 64, 48, 64), 5).to(DEV)
    loss = head(x).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        loss.backward()
    loss = head(x).sum()
    with torch.no_grad():
        head[0].project[0].weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()
    xg = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(head(xg).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


def test_encoder_heads_stay_eval_only():
    head = make_head(160, 160, 64).to(DEV)
    from stp3_b200 import dense
    with pytest.raises(NotImplementedError, match="call .eval()"):
        head.forward_hl(dense.from_f32(gauss((2, 1, 160, 14, 30), 5).to(DEV)))


# ------------------------------------------------------------------------------------------------ model level
def small_stp3():
    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    from stp3_b200.utils import geometry as Geo
    from stp3_b200.utils import synthetic as syn
    cfg = get_cfg({"LIFT": {"X_BOUND": [-8.0, 8.0, 0.5], "Y_BOUND": [-8.0, 8.0, 0.5], "D_BOUND": [2.0, 10.0, 1.0]},
                   "IMAGE": {"FINAL_DIM": (32, 48)}})
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
    inp = syn.lift_inputs(lcfg, 2, seed=4, random_pose=True)
    model = STP3(cfg, backbone=torch.nn.Identity())
    with torch.no_grad():
        TD.init_exact(model, seed=7)
        model.frustum.copy_(model.create_frustum())
        res, start, dim = Geo.calculate_birds_eye_view_parameters(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND)
        model.bev_resolution.copy_(res); model.bev_start_position.copy_(start); model.bev_dimension.copy_(dim)
    return model.to(DEV), inp


def test_recipe_trains_head_and_decoder():
    from stp3_b200.models.stp3 import GraphedPerception
    model, inp = small_stp3()
    model.eval()
    head = model.temporal_model.final_conv
    head.train()
    fwd = lambda: model.forward_features(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],  # noqa
                                         inp["extrinsics"], inp["future_egomotion"])
    with pytest.raises(RuntimeError, match="decoder is in eval mode"):
        fwd()
    with pytest.raises(RuntimeError, match="final_conv is in train mode"):
        GraphedPerception(model, 2, 2)
    model.decoder.train()
    # the head's input: the eval-mode TemporalBlocks on the BEV grid, captured on the way in
    seen = {}
    hook = head.register_forward_pre_hook(lambda m, a: seen.setdefault("x", a[0].detach().clone()))
    ref_head = copy.deepcopy(head).double()
    ref_dec = copy.deepcopy(model.decoder).double()
    before = {k: b.clone() for k, b in model.named_buffers()}
    torch.manual_seed(21)
    out = fwd()
    hook.remove()
    keys = ("segmentation", "pedestrian", "hdmap")
    loss = sum(out[k].float().square().mean() for k in keys)
    loss.backward()
    for k, p in model.named_parameters():
        trained = k.startswith("temporal_model.final_conv.") or k.startswith("decoder.")
        assert (p.grad is not None) == trained, k
        if trained:
            assert torch.isfinite(p.grad).all(), k
    for k, b in model.named_buffers():
        if "running" in k or "num_batches" in k:
            trained = k.startswith("temporal_model.final_conv.") or k.startswith("decoder.")
            assert (not torch.equal(b, before[k])) == trained, k
    # fp64: the train-mode head (its native dropout mask and ReLU branches pinned) then the train-mode decoder
    x = seen["x"]
    masks, keep = native_masks(copy.deepcopy(ref_head).float().cpu(), x.cpu(), seed=21)
    queue = list(masks)
    y = TH.deeplab_head_train(x.double(), ref_head.to(DEV), relu=lambda t: t * queue.pop(0),
                              dropout_mask=keep.permute(0, 3, 1, 2))
    B, S = 2, model.receptive_field
    want = TT.decoder_train(y.view(B, S, *y.shape[1:]), ref_dec.to(DEV))
    for k in keys:
        e = rel_max(out[k].detach(), want[k].detach())
        assert e < 1e-3, (k, e)
