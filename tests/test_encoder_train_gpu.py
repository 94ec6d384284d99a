"""GPU: the encoder heads in train mode on the sm_90a kernels.

Kernel level: the channel-window bilinear x2 pair against fp64 F.interpolate and its adjoint, and bitwise against the
dense entry points; stp3_lift_splat_bwd_cl bitwise against stp3_lift_splat_bwd on transposed tensors and against the fp64
oracle.  Module level: UpsamplingConcat and one encoder head (DeepLabHead -> UpsamplingConcat) -- outputs, running
statistics and every gradient against fp64 autograd through oracle/torch_encoder_train with the ReLU branches and the
dropout mask pinned to the native forward, against the reference fixture, determinism, a train step followed by an eval
forward, the autograd guards, the refusals.  Model level: the three recipes (trunk endpoints that require grad, an
injected torch trunk under model.train(), the frozen native trunk with train_heads())."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet_oracle as EO
from oracle import lift_splat_oracle as O
from oracle import make_golden_encoder_train as MG
from oracle import torch_dense as TD
from oracle import torch_dense_train as TT
from oracle import torch_encoder_train as TE
from oracle.make_golden_bwd import loss_weights
from stp3_b200 import dense_train as T
from stp3_b200 import ops
from stp3_b200.layers import convolutions as CV
from stp3_b200.utils import geometry as G
from stp3_b200.utils import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rel_max(got, ref):
    got, ref = got.double(), ref.double().to(got.device)
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def nchw(t):
    return t.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("cf,cc", [(56, 160), (40, 112), (3, 5)])
def test_channel_window_upsample_pair(cf, cc):
    N, h, w = 3, 14, 30
    x = gauss((N, h, w, cc), 1).to(DEV)
    cat = torch.full((N, 2 * h, 2 * w, cf + cc), float("nan"), device=DEV)
    T.upsample2x_into(x, cat, cf)
    x64 = nchw(x).double().requires_grad_(True)
    ref = F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=False)
    assert torch.isnan(cat[..., :cf]).all()                        # the fine map's channels are not touched
    assert rel_max(nchw(cat[..., cf:]), ref.detach()) < 1e-6
    # the window form (16-byte or scalar accesses, strided rows) stores the dense entry point's values
    assert torch.equal(cat[..., cf:], T.upsample2x(x))
    gy = gauss((N, 2 * h, 2 * w, cf + cc), 2).to(DEV)
    gx = T.upsample2x_backward_from(gy, cf, cc)
    ref.backward(nchw(gy[..., cf:]).double())
    assert rel_max(nchw(gx), x64.grad) < 1e-6
    assert torch.equal(gx, T.upsample2x_backward(gy[..., cf:].contiguous()))
    assert torch.equal(gx, T.upsample2x_backward_from(gy, cf, cc))


SMALL = dict(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0), n_cameras=2, receptive_field=3)
LIFT_CASES = {
    "plumbing_depth": (syn.CONFIGS["plumbing"], 1, False, True),
    "plumbing_b2_no_depth": (syn.CONFIGS["plumbing"], 2, True, False),
    "lift_splat": (syn.CONFIGS["lift_splat"], 1, True, True),
    "ragged_width": (syn.LiftSplatConfig(final_dim=(32, 80), out_channels=64, **SMALL), 1, True, True),     # Wf = 10
    "two_channel_passes": (syn.LiftSplatConfig(final_dim=(32, 48), out_channels=128, **SMALL), 2, True, True),
}


@pytest.mark.parametrize("name", list(LIFT_CASES))
def test_lift_splat_backward_channels_last_equals_nchw_bitwise(name):
    cfg, batch, rp, use_dd = LIFT_CASES[name]
    inp = syn.lift_inputs(cfg, batch, seed=21, random_pose=rp)
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(cfg.final_dim, cfg.downsample, cfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
    off = G.bev_offset(start, res)
    geo = (cam_M, cam_t, ego_R, ego_t, xs, ys, ds, off, res, dim, cfg.discount)
    feat, depth = inp["feat"].to(DEV), inp["depth_logits"].to(DEV)
    feat_cl = feat.permute(0, 1, 2, 4, 5, 3).contiguous()
    out, ranks = ops.lift_splat(feat, depth, *geo, use_depth_distribution=use_dd, return_ranks=True)
    W = loss_weights(tuple(out.shape), 5)
    gf, gd = ops.lift_splat_backward(W.to(DEV), feat, depth, *geo, use_depth_distribution=use_dd)
    gf_cl, gd_cl = ops.lift_splat_backward(W.to(DEV), feat_cl, depth, *geo, use_depth_distribution=use_dd,
                                           feat_channels_last=True)
    torch.cuda.synchronize()
    assert gf_cl.shape == feat_cl.shape
    assert torch.equal(gf_cl.permute(0, 1, 2, 5, 3, 4), gf)
    assert (gd is None and gd_cl is None) if not use_dd else torch.equal(gd_cl, gd)
    ogf, ogd = O.lift_splat_backward(W.numpy(), inp["feat"].numpy(), inp["depth_logits"].numpy(), ranks.cpu().numpy(),
                                     cfg.discount, use_depth_distribution=use_dd)
    assert np.abs(gf_cl.permute(0, 1, 2, 5, 3, 4).double().cpu().numpy() - ogf).max() <= 1e-5 * np.abs(ogf).max()
    if use_dd:
        assert np.abs(gd_cl.double().cpu().numpy() - ogd).max() <= 1e-5 * np.abs(ogd).max()
    # through autograd: the gradient of channels-last features comes back channels-last
    f = feat_cl.clone().requires_grad_(True)
    d = depth.clone().requires_grad_(use_dd)
    bev = ops.lift_splat_autograd(f, d, *geo, use_depth_distribution=use_dd, feat_channels_last=True)
    assert rel_max(bev.detach(), out) < 1e-5          # the forward's float atomics: summation order only
    (bev * W.to(DEV)).sum().backward()
    assert torch.equal(f.grad, gf_cl) and (not use_dd or torch.equal(d.grad, gd_cl))


# ------------------------------------------------------------------------------------------------ module level
def modules(name, momentum=MG.MOMENTUM):
    head, up, mods = MG.make_modules(CV, name)
    for m in mods.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = momentum
    return head, up, mods


def native_forward(head, up, r_lo, r_hi, seed=None):
    """The native train forward on copies -> (ReLU masks in the restatement's call order, dropout keep mask or None).
    seed None: the dropout seed is the next draw of torch's generator, as in a forward that ran other heads before."""
    head, up = copy.deepcopy(head), copy.deepcopy(up).to(DEV)
    masks, keep, x_up = [], None, r_hi.to(DEV)
    if seed is not None:
        torch.manual_seed(seed)
    with torch.no_grad():
        if head is not None:
            x_up, t = head.to(DEV)._train_forward(x_up)
            h = head.hidden
            masks = [nchw(t["cat"][..., i * h:(i + 1) * h] > 0).double() for i in range(len(t["branches"]))]
            masks += [nchw(t[k] > 0).double() for k in ("v", "z", "y3")]
            keep = nchw(t["z"] != 0)
        _, t = up._train_forward(x_up, r_lo.to(DEV), False)
    return masks + [nchw(t["y0"] > 0).double(), nchw(t["y1"] > 0).double()], keep


def oracle_step(head, up, r_lo, r_hi, Gout, masks, keep):
    mods = copy.deepcopy(torch.nn.ModuleList([m for m in (head, up) if m is not None])).double().to(DEV)
    lo = r_lo.double().to(DEV).requires_grad_(True)
    hi = r_hi.double().to(DEV).requires_grad_(True)
    queue = list(masks)
    relu = lambda t: t * queue.pop(0)        # noqa: E731
    if head is None:
        out = TE.upsampling_concat_train(hi, lo, mods[0], relu=relu)
    else:
        out = TE.encoder_head_train(lo, hi, mods[0], mods[1], relu=relu, dropout_mask=keep)
    assert not queue
    (out * Gout.double().to(DEV)).sum().backward()
    return out.detach(), mods, lo.grad, hi.grad


def native_step(head, up, r_lo, r_hi, Gout, seed, channels_last=False):
    lo, hi = r_lo.to(DEV).requires_grad_(True), r_hi.to(DEV).requires_grad_(True)
    for m in (head, up):
        if m is not None:
            m.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    out = up(head(hi) if head is not None else hi, lo, channels_last=channels_last)
    Gd = Gout.to(DEV)
    (out * (Gd.permute(0, 2, 3, 1) if channels_last else Gd)).sum().backward()
    torch.cuda.synchronize()
    return out, lo.grad, hi.grad


@pytest.mark.parametrize("name", ["uc", "feat", "depth"])
def test_train_step_matches_fp64_oracle_and_reference_fixture(name):
    head, up, mods = modules(name)
    r_lo, r_hi = MG.endpoints()
    cout = up.out_channels
    Gout = TT.upstream_grads({"out": torch.empty(MG.M, cout, 2 * MG.H, 2 * MG.W)}, seed=MG.GRAD_SEED)["out"]
    masks, keep = native_forward(head, up, r_lo, r_hi, seed=17)
    out_ref, ref, glo_ref, ghi_ref = oracle_step(head, up, r_lo, r_hi, Gout, masks, keep)
    mods = mods.to(DEV)
    out, glo, ghi = native_step(head, up, r_lo, r_hi, Gout, seed=17)
    assert out.grad_fn is not None and tuple(out.shape) == (MG.M, cout, 2 * MG.H, 2 * MG.W)
    worst = {"out": rel_max(out.detach(), out_ref), "grad.r_lo": rel_max(glo, glo_ref), "grad.r_hi": rel_max(ghi, ghi_ref)}
    for (k, b), (_, b_ref) in zip(mods.named_buffers(), ref.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(b_ref) == 1, k
            continue
        assert rel_max(b, b_ref) < 1e-5, k
    for (k, p), (_, p_ref) in zip(mods.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, f"{k}: no gradient"
        worst[f"grad.{k}"] = rel_max(p.grad, p_ref.grad)
    print(name, sorted(((k, f"{v:.2e}") for k, v in worst.items()), key=lambda kv: -float(kv[1]))[:4])
    bad = {k: v for k, v in worst.items() if v > 1e-3}
    assert not bad, bad
    # the reference's own fp32 UpsamplingConcat: output and running statistics.  Its gradients depend on ReLU branches
    # of inputs within round-off of zero; tests/test_encoder_train_cpu.py ties them to the fp64 oracle used above with
    # those branches pinned
    if name == "uc":
        golden = np.load("tests/golden/encoder_heads_train.npz")
        flat = out.detach().reshape(-1).cpu()
        s = golden["uc.out_s"]
        e = np.abs(flat[TT.sample_index("uc.out", flat.numel(), len(s))].numpy() - s).max() / golden["uc.out_amax"]
        assert e < 1e-3, e
        for k, b in mods.named_buffers():
            if not k.endswith("num_batches_tracked"):
                assert rel_max(b, torch.from_numpy(golden["uc." + k])) < 1e-4, k
    # two runs are bitwise equal, and the channels-last form is the same numbers transposed
    grads1 = [p.grad.clone() for p in mods.parameters()]
    out2, glo2, ghi2 = native_step(head, up, r_lo, r_hi, Gout, seed=17)
    assert torch.equal(out, out2) and torch.equal(glo, glo2) and torch.equal(ghi, ghi2)
    assert all(torch.equal(a, p.grad) for a, p in zip(grads1, mods.parameters()))
    out3, glo3, ghi3 = native_step(head, up, r_lo, r_hi, Gout, seed=17, channels_last=True)
    assert torch.equal(out3.permute(0, 3, 1, 2), out) and torch.equal(glo, glo3) and torch.equal(ghi, ghi3)
    assert all(torch.equal(a, p.grad) for a, p in zip(grads1, mods.parameters()))


def test_gradients_only_where_required():
    _, up, mods = modules("uc")
    mods.to(DEV)
    r_lo, r_hi = (t.to(DEV) for t in MG.endpoints())
    up(r_hi, r_lo.requires_grad_(True)).sum().backward()
    assert r_lo.grad is not None and r_hi.grad is None
    with torch.no_grad():
        assert up(r_hi, r_lo).grad_fn is None


def test_sgd_step_then_eval_matches_eval_oracle():
    _, up, mods = modules("uc", momentum=0.1)
    mods.to(DEV)
    r_lo, r_hi = (t.to(DEV) for t in MG.endpoints())
    up.eval()
    with torch.no_grad():
        up(r_hi, r_lo)                              # packs (and caches) the eval-mode weights
    up.train()
    opt = torch.optim.SGD(up.parameters(), lr=0.05)
    (up(r_hi, r_lo) ** 2).mean().backward()
    opt.step()
    up.eval()
    with torch.no_grad():
        got = up(r_hi, r_lo)
        m64 = copy.deepcopy(up).cpu().double()
        y = torch.cat([r_lo.double().cpu(), F.interpolate(r_hi.double().cpu(), scale_factor=2, mode="bilinear",
                                                          align_corners=False)], 1)
        ref = m64.conv(y)                           # plain nn modules in eval mode: the folded weights' meaning
    assert rel_max(got, ref) < 1e-3


def test_autograd_node_guards():
    _, up, mods = modules("uc")
    mods.to(DEV)
    r_lo, r_hi = (t.to(DEV) for t in MG.endpoints())
    loss = up(r_hi, r_lo).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        loss.backward()
    loss = up(r_hi, r_lo).sum()
    with torch.no_grad():
        up.conv[3].weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()
    xg = r_lo.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(up(r_hi, xg).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


@pytest.mark.parametrize("what", ["sync", "momentum_none", "no_running_stats", "shape"])
def test_refusals(what):
    _, up, mods = modules("uc")
    r_lo, r_hi = (t.to(DEV) for t in MG.endpoints())
    exc = NotImplementedError
    if what == "sync":
        up, match = torch.nn.SyncBatchNorm.convert_sync_batchnorm(up), "SyncBatchNorm"
    elif what == "momentum_none":
        up.conv[1].momentum, match = None, "momentum=None"
    elif what == "no_running_stats":
        up.conv[4].track_running_stats, match = False, "track_running_stats=False"
    else:
        r_lo, exc, match = r_lo[..., :-2], ValueError, "expected"
    with pytest.raises(exc, match=match):
        up.to(DEV).train()(r_hi, r_lo)


# ------------------------------------------------------------------------------------------------ model level
LCFG = syn.LiftSplatConfig(final_dim=(128, 192), out_channels=64, **SMALL)


class ConvTrunk(torch.nn.Module):
    """A small torch trunk with the encoder's endpoint shapes: (M,3,H,W) -> ((M,56,H/8,W/8), (M,160,H/16,W/16))."""

    def __init__(self):
        super().__init__()
        self.a = torch.nn.Conv2d(3, 56, 8, stride=8)
        self.b = torch.nn.Conv2d(56, 160, 2, stride=2)

    def forward(self, x):
        r3 = F.relu(self.a(x))
        return r3, F.relu(self.b(r3))


def small_stp3(backbone):
    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    cfg = get_cfg({"LIFT": {"X_BOUND": list(LCFG.x_bound), "Y_BOUND": list(LCFG.y_bound), "D_BOUND": list(LCFG.d_bound)},
                   "IMAGE": {"FINAL_DIM": LCFG.final_dim}})
    model = STP3(cfg, backbone=backbone)
    with torch.no_grad():
        geo = {k: getattr(model, k).detach().clone() for k in ("frustum", "bev_resolution", "bev_start_position", "bev_dimension")}
        trunk = copy.deepcopy(model.encoder.backbone.state_dict())
        TD.init_exact(model, seed=7)
        for k, v in geo.items():
            getattr(model, k).copy_(v)
        model.encoder.backbone.load_state_dict(trunk)
    return model.to(DEV), syn.lift_inputs(LCFG, 1, seed=4, random_pose=True)


def loss_of(out):
    return sum(out[k].float().square().mean() for k in ("segmentation", "pedestrian", "hdmap")) + \
        out["depth_prediction"].float().square().mean() * 0.01


def check_refused_by_graph_and_sharded(model, inp):
    from stp3_b200.models.stp3 import GraphedPerception
    for entry in ("lift", "heads"):
        with pytest.raises(RuntimeError, match="train mode"):
            GraphedPerception(model, 1, 2, entry=entry)
    with pytest.raises(RuntimeError, match="encoder heads are in train mode"):
        model.forward_features_frame_sharded(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                             inp["extrinsics"], inp["future_egomotion"])


def test_endpoints_that_require_grad_train_everything_behind_the_trunk():
    model, inp = small_stp3(torch.nn.Identity())
    B, S, N = 1, 3, 2
    Hf, Wf = LCFG.feat_hw
    r_lo = gauss((B, S, N, 56, Hf, Wf), 1).to(DEV).requires_grad_(True)
    r_hi = gauss((B, S, N, 160, Hf // 2, Wf // 2), 2).to(DEV).requires_grad_(True)
    fwd = lambda: model.forward_trunk_features(r_lo, r_hi, inp["intrinsics"], inp["extrinsics"],   # noqa: E731
                                               inp["future_egomotion"])
    model.eval()
    enc = model.encoder
    enc.train_heads()
    with pytest.raises(RuntimeError, match="call model.temporal_model.train"):
        fwd()
    model.temporal_model.train()
    model.decoder.train()
    check_refused_by_graph_and_sharded(model, inp)
    # the gradients that arrive at the two heads' outputs, and the heads' modules as they were before the step
    before = {k: copy.deepcopy(getattr(enc, k)) for k in ("feature_layer_1", "feature_layer_2", "depth_layer_1",
                                                          "depth_layer_2")}
    seen = {}
    inner = enc.heads_train

    def spy(lo, hi, channels_last=False):
        feat, depth = inner(lo, hi, channels_last)
        assert channels_last and feat.shape[-1] == 64
        feat.register_hook(lambda g: seen.__setitem__("g_feat", g.detach().clone()))
        depth.register_hook(lambda g: seen.__setitem__("g_depth", g.detach().clone()))
        return feat, depth
    enc.heads_train = spy
    torch.manual_seed(31)
    out = fwd()
    assert out["depth_prediction"].grad_fn is not None and tuple(out["depth_prediction"].shape) == (B, S, N, 8, Hf, Wf)
    loss_of(out).backward()
    torch.cuda.synchronize()
    for k, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
            assert not k.startswith("encoder.") or p.grad.abs().max() > 0, k
    # fp64: both heads with the native masks, driven by the gradients that arrived; their input gradients add up
    lo2, hi2 = r_lo.detach().flatten(0, 2).cpu(), r_hi.detach().flatten(0, 2).cpu()
    pairs = (("feature_layer_1", "feature_layer_2", nchw(seen["g_feat"])),
             ("depth_layer_1", "depth_layer_2", seen["g_depth"]))
    torch.manual_seed(31)                 # the forward drew the feature head's dropout seed, then the depth head's
    pinned = [native_forward(before[l1].cpu(), before[l2].cpu(), lo2, hi2) for l1, l2, _ in pairs]
    want_lo = want_hi = 0
    for (l1, l2, g), (masks, keep) in zip(pairs, pinned):
        _, ref, glo, ghi = oracle_step(before[l1].cpu(), before[l2].cpu(), lo2, hi2, g, masks, keep)
        want_lo, want_hi = want_lo + glo, want_hi + ghi
        got = list(getattr(enc, l1).named_parameters()) + list(getattr(enc, l2).named_parameters())
        for (k, p), (_, p_ref) in zip(got, ref.named_parameters()):
            e = rel_max(p.grad, p_ref.grad)
            assert e < 1e-3, (l1, k, e)
    assert rel_max(r_lo.grad.flatten(0, 2), want_lo) < 1e-3
    assert rel_max(r_hi.grad.flatten(0, 2), want_hi) < 1e-3


def test_reference_recipe_trains_an_injected_torch_trunk():
    model, inp = small_stp3(ConvTrunk())
    model.train()
    image = gauss((1, 3, 2, 3, *LCFG.final_dim), 3).to(DEV)
    check_refused_by_graph_and_sharded(model, inp)
    out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    loss_of(out).backward()
    torch.cuda.synchronize()
    for k, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
            assert not k.startswith("encoder.") or p.grad.abs().max() > 0, k
    assert model.encoder.backbone.a.weight.grad is not None


def test_frozen_native_trunk_recipe():
    model, inp = small_stp3("native")
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=5), 'b4').eval()
    model.encoder.backbone.load_state_dict(ora.state_dict(), strict=True)
    model = model.to(DEV)
    with pytest.raises(NotImplementedError, match="eval-mode forward only"):
        model.train()
    model.eval()
    model.encoder.train_heads()
    model.temporal_model.train()
    model.decoder.train()
    image = gauss((1, 3, 2, 3, *LCFG.final_dim), 3).to(DEV)
    trunk_state = {k: v.clone() for k, v in model.encoder.backbone.state_dict().items()}
    out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    loss_of(out).backward()
    torch.cuda.synchronize()
    for k, p in model.named_parameters():
        if k.startswith("encoder.backbone."):
            assert p.grad is None, k
        elif p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
    assert all(torch.equal(v, trunk_state[k]) for k, v in model.encoder.backbone.state_dict().items())
    for k, b in model.named_buffers():
        if k.endswith("num_batches_tracked") and not k.startswith("encoder.backbone."):
            assert int(b) == 1, k
