"""GPU: the TemporalBlocks in train mode (batch statistics, causal 3-D convolution gradients, the pyramid-pooling branch
over the batch, autograd) on the sm_90a kernels.

Kernel level: causal 3-D weight / input gradients against fp64 torch autograd (time taps that read only padding give
exact zeros), BatchNorm at channel counts that are not multiples of 8 against fp64, and the vector BatchNorm path bitwise
equal to checksums recorded with the library before the scalar path existed.  Module level: TemporalModel (blocks and
head in train mode) against fp64 autograd through oracle/torch_temporal_train with the ReLU branches and the head's
dropout mask pinned to the native forward; determinism, a train step followed by an eval forward, the no-grad
running-statistics update, the refusals.  Model level: the recipe model.train(); model.encoder.eval() on a small STP3."""
import copy
import hashlib

import pytest
import torch
import torch.nn.functional as F

from oracle import torch_dense as TD
from oracle import torch_dense_train as TT
from oracle import torch_temporal_train as OT
from stp3_b200 import _lib, dense, dense_train as T
from stp3_b200.models.temporal_model import TemporalModel, _TemporalBlocksTrainFn
from tests.test_deeplab_train_gpu import native_masks as head_masks, small_stp3
from tests.test_decoder_train_gpu import native_relu_masks as dec_masks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gauss(shape, seed):
    return TD.exact_gauss(shape, torch.Generator().manual_seed(seed))


def rel_max(got, ref):
    got, ref = got.double(), ref.double().to(got.device)
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def causal_conv3d(x, w):
    kt, kh, kw = w.shape[2:]
    return F.conv3d(F.pad(x, ((kw - 1) // 2, (kw - 1) // 2, (kh - 1) // 2, (kh - 1) // 2, kt - 1, 0)), w)


# ------------------------------------------------------------------------------------------------ kernel level
GEOMS = [(48, 64, 3, 2), (48, 64, 5, 1), (200, 200, 3, 2), (200, 200, 5, 1)]


@pytest.mark.parametrize("c", [35, 32, 67])
@pytest.mark.parametrize("k", [(2, 3, 3), (1, 3, 3), (1, 1, 1)])
@pytest.mark.parametrize("geom", GEOMS)
def test_conv3d_wgrad_dgrad(c, k, geom):
    H, W, t, B = geom
    x = gauss((B, c, t, H, W), 1).double().to(DEV).requires_grad_(True)
    w = (gauss((c, c, *k), 2).double() * 0.05).to(DEV).requires_grad_(True)
    g = gauss((B, c, t, H, W), 3).double().to(DEV)
    dx_ref, dw_ref = torch.autograd.grad(causal_conv3d(x, w), (x, w), g)
    x_cl = x.detach().float().permute(0, 2, 3, 4, 1).contiguous()
    g_cl = g.float().permute(0, 2, 3, 4, 1).contiguous()
    dw = T.conv_wgrad(x_cl, g_cl, k[1], k[2], 1, kt=k[0])
    dx = T.conv_dgrad(g_cl.view(B * t, H, W, c), w.detach().float(), 1, H, W, T=t)
    torch.cuda.synchronize()
    e_w = rel_max(dw, dw_ref)
    e_x = rel_max(dx.view(B, t, H, W, c).permute(0, 4, 1, 2, 3), dx_ref)
    print(f"{k} {c}->{c} B{B} T{t} {H}x{W}: wgrad {e_w:.2e}, dgrad {e_x:.2e} of max")
    assert e_w < 1e-3 and e_x < 1e-3, (e_w, e_x)
    assert torch.equal(dw, T.conv_wgrad(x_cl, g_cl, k[1], k[2], 1, kt=k[0]))


def test_conv3d_wgrad_all_padding_time_tap_is_exact_zero():
    B, t, H, W, c = 2, 1, 48, 64, 35
    x = gauss((B, t, H, W, c), 1).to(DEV)
    g = gauss((B, t, H, W, c), 3).to(DEV)
    dw = T.conv_wgrad(x, g, 3, 3, 1, kt=2)
    assert not dw[:, :, 0].any()                     # frame t - 1 is padding for every output frame
    ref = T.conv_wgrad(x.view(B * t, H, W, c), g.view(B * t, H, W, c), 3, 3, 1)
    assert torch.equal(dw[:, :, 1], ref)             # the present-frame tap is the 2-D weight gradient, bit for bit


@pytest.mark.parametrize("C", [21, 23, 35, 44, 67])
def test_batchnorm_any_channel_count(C):
    n_img, H, W = 6, 48, 64
    wide = gauss((n_img, H, W, C + 5), 4).to(DEV) * 2.0 + 0.5
    x = wide[..., 3:3 + C]                           # a channel window at an odd offset: no 16-byte rows
    gamma, beta = (gauss((C,), 5) * 0.3 + 1.0).to(DEV), (gauss((C,), 6) * 0.1).to(DEV)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    xc = x.contiguous()
    st = T.bn_stats(xc, 1e-5, 0.1, rm, rv)
    out = torch.empty((n_img, H, W, C + 3), device=DEV)
    y, y_hl = T.bn_apply(xc, st, gamma, beta, relu=True, y_out=out[..., 1:1 + C])
    xd = x.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
    bn = torch.nn.BatchNorm2d(C, momentum=0.1).double()
    with torch.no_grad():
        bn.weight.copy_(gamma.cpu()); bn.bias.copy_(beta.cpu())
    yd = F.relu(bn(xd))
    assert rel_max(y.permute(0, 3, 1, 2), yd) < 1e-5
    assert rel_max(dense.to_f32(dense.HL(y_hl.hi, y_hl.lo, C)).squeeze(1), yd) < 1e-5
    assert not y_hl.hi[..., C:].any() and not y_hl.lo[..., C:].any()
    assert rel_max(rm, bn.running_mean) < 1e-6 and rel_max(rv, bn.running_var) < 1e-6
    g = gauss((n_img, H, W, C), 7).to(DEV)
    dx_full = torch.zeros((n_img, H, W, C + 2), device=DEV)
    dx, dgam, dbet, gm = T.bn_backward(g, xc, st, gamma, y, want_masked=True, dx_out=dx_full[..., 2:])
    (gx, gg, gb) = torch.autograd.grad(yd, (xd, bn.weight, bn.bias), g.double().cpu().permute(0, 3, 1, 2))
    assert rel_max(dx.permute(0, 3, 1, 2), gx) < 1e-4
    assert rel_max(dgam, gg) < 1e-5 and rel_max(dbet, gb) < 1e-5
    assert torch.equal(gm, torch.where(y > 0, g, torch.zeros_like(g)))
    assert not dx_full[..., :2].any()


def bn_vector_outputs(L):
    """sha256 prefixes of stp3_bn_apply / stp3_bn_bwd_apply outputs on inputs the vector path accepts (C % 8 == 0,
    16-byte rows; residual, dropout, bf16 planes, masks), through the library handle L."""
    s = torch.cuda.current_stream().cuda_stream
    out = {}
    for C, cs in ((64, 64), (128, 136), (8, 8)):
        n = 6 * 48 * 64
        x = gauss((n, cs), 11).to(DEV)
        res = gauss((n, cs), 12).to(DEV)
        mean, invstd = (gauss((C,), 13) * 0.1).to(DEV), (gauss((C,), 14).abs() + 0.5).to(DEV)
        gam, bet = (gauss((C,), 15) + 1.0).to(DEV), (gauss((C,), 16) * 0.1).to(DEV)
        for p, use_res in ((0.0, False), (0.5, True)):
            y = torch.zeros((n, cs), device=DEV)
            hi = torch.zeros((n, 128 if C <= 128 else 192), dtype=torch.bfloat16, device=DEV)
            lo = torch.zeros_like(hi)
            rc = L.stp3_bn_apply(x.data_ptr(), n, C, cs, mean.data_ptr(), invstd.data_ptr(), gam.data_ptr(),
                                 bet.data_ptr(), res.data_ptr() if use_res else None, cs, 1, p, 77, 5,
                                 y.data_ptr(), cs, hi.data_ptr(), lo.data_ptr(), hi.shape[1], s)
            assert rc == 0
            torch.cuda.synchronize()
            out[("apply", C, p)] = sha(y) + sha(hi) + sha(lo)
        g = gauss((n, cs), 17).to(DEV)
        sg, sgx = (gauss((C,), 18) * 10).to(DEV), (gauss((C,), 19) * 10).to(DEV)
        dx = torch.zeros((n, cs), device=DEV)
        gm = torch.zeros((n, cs), device=DEV)
        rc = L.stp3_bn_bwd_apply(g.data_ptr(), cs, res.data_ptr(), cs, x.data_ptr(), cs, mean.data_ptr(),
                                 invstd.data_ptr(), gam.data_ptr(), sg.data_ptr(), sgx.data_ptr(), n, C, dx.data_ptr(),
                                 cs, gm.data_ptr(), cs, s)
        assert rc == 0
        torch.cuda.synchronize()
        out[("bwd", C)] = sha(dx) + sha(gm)
    return out


def sha(t):
    return hashlib.sha256(t.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()[:12]


# recorded with the library before stp3_bn_apply / stp3_bn_bwd_apply had a scalar path (H100 80GB HBM3, 700 W)
BN_VECTOR_SHA = {
    ("apply", 64, 0.0): "e389cd9bac376f1facb12d9d1b70cd39eacd", ("apply", 64, 0.5): "ee10d967bc07834f658d1d341a7e0472a332",
    ("bwd", 64): "5774c2c5c4187ab4e7e65060",
    ("apply", 128, 0.0): "5e3e01a068e3c7524abf5ef2cc1133dba6eb", ("apply", 128, 0.5): "d536e01f0979006a056c8fa1e18a101ecafb",
    ("bwd", 128): "8228aaa7ccc5382ca0416003",
    ("apply", 8, 0.0): "ab098f401ed412fcb2e8838843e86af71b69", ("apply", 8, 0.5): "5bc844bf79a617bdbeb75b0bcf6171f18a9d",
    ("bwd", 8): "a59442868fd635a35cf31114",
}


def test_batchnorm_vector_path_bitwise_unchanged():
    assert bn_vector_outputs(_lib.lib()) == BN_VECTOR_SHA


def test_pair_mean_kernel():
    B, t, C = 2, 5, 70
    m = gauss((B * t, C), 8).to(DEV)
    p = T.temporal_pair_mean(m, t)
    assert rel_max(p, OT.pair_mean(m.double(), t)) < 1e-6
    g = gauss((B * (t + 1), C), 9).to(DEV)
    md = m.double().requires_grad_(True)
    (ref,) = torch.autograd.grad(OT.pair_mean(md, t), md, g.double())
    assert rel_max(T.temporal_pair_mean(g, t, adjoint=True), ref) < 1e-6


# ------------------------------------------------------------------------------------------------ module level
# name -> (in_channels (with the constant ones), n_const, S, B, H, W)
CONFIGS = {"perceive_48x64": (70, 0, 3, 2, 48, 64), "perceive_ego_48x64": (70, 6, 3, 2, 48, 64),
           "perceive_ego_200x200": (70, 6, 3, 2, 200, 200), "stress_16x24": (134, 0, 5, 1, 16, 24)}


def make_model(cin, nc, S, H, W, momentum=0.05):
    tm = TD.init_exact(TemporalModel(cin, S, (H, W), start_out_channels=64), seed=3)
    for m in tm.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = momentum
    if len(tm.model):
        tm.model[0].n_const = nc
    return tm.train()


def inputs(cin, nc, S, B, H, W):
    x = gauss((B, S, cin - nc, H, W), 5)
    const = gauss((B * S, nc), 6) if nc else None
    return x, const


def full_input(x, const):
    """x with the constant channels broadcast behind it: what the reference model sees."""
    if const is None:
        return x
    B, S, _, H, W = x.shape
    return torch.cat([x, const.view(B, S, -1, 1, 1).expand(B, S, const.shape[1], H, W)], 2)


def native_masks(tm_cpu, x, const, seed):
    """(ReLU masks of the blocks and the head in the restatement's call order, head dropout keep mask) of the native
    forward, as fp64 tensors in the reference layouts."""
    tm = copy.deepcopy(tm_cpu).to(DEV)
    B, S, C, H, W = x.shape
    masks = []
    with torch.no_grad():
        y = x.to(DEV).permute(0, 1, 3, 4, 2).reshape(B * S, H, W, C).contiguous()
        c = const.to(DEV) if const is not None else None
        ncdhw = lambda t: (t > 0).reshape(B, -1, *t.shape[1:]).permute(0, 4, 1, 2, 3).double()   # noqa: E731
        for i, blk in enumerate(tm.model):
            y, tape = blk._train_forward(y, c if i == 0 else None, B, S)
            h = blk.half_channels
            cat = tape["cat"]
            masks += [ncdhw(tape["entry"][0][3]), ncdhw(cat[..., :h]), ncdhw(tape["entry"][1][3]),
                      ncdhw(cat[..., h:2 * h]), ncdhw(cat[..., 2 * h:])]
            if blk.use_pyramid_pooling:
                masks.append(ncdhw(tape["v_full"]))
            masks.append(ncdhw(tape["ya"]))
    hm, keep = head_masks(copy.deepcopy(tm_cpu.final_conv), y.permute(0, 3, 1, 2).cpu(), seed)
    return masks + hm, keep


def oracle_step(tm_cpu, x, const, G, masks, keep):
    ref = copy.deepcopy(tm_cpu).double().to(DEV)
    xd = full_input(x, const).double().to(DEV).requires_grad_(True)
    queue = list(masks)
    out = OT.temporal_model_train(xd, ref, relu=lambda t: t * queue.pop(0), dropout_mask=keep.permute(0, 3, 1, 2))
    assert not queue
    (out * G.double().to(DEV)).sum().backward()
    return out, ref, xd.grad[:, :, :x.shape[2]]


def native_step(tm, x, const, G, seed):
    x = x.to(DEV).requires_grad_(True)
    tm.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    out = tm(x, const=const.to(DEV) if const is not None else None)
    (out * G.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    return out, x.grad


@pytest.mark.parametrize("name", list(CONFIGS))
def test_train_step_matches_fp64_oracle(name):
    cin, nc, S, B, H, W = CONFIGS[name]
    tm_cpu = make_model(cin, nc, S, H, W)
    x, const = inputs(cin, nc, S, B, H, W)
    G = gauss((B, S, 64, H, W), 9) * 0.25
    masks, keep = native_masks(tm_cpu, x, const, seed=17)
    out_ref, ref, gx_ref = oracle_step(tm_cpu, x, const, G, masks, keep)
    tm = copy.deepcopy(tm_cpu).to(DEV)
    out, gx = native_step(tm, x, const, G, seed=17)
    assert out.grad_fn is not None
    worst = {"out": rel_max(out.detach(), out_ref.detach())}
    for (k, b), (_, b_ref) in zip(tm.named_buffers(), ref.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(b_ref) == 1, k
            continue
        e = rel_max(b, b_ref)
        assert e < 1e-5, (k, e)
    for (k, p), (_, p_ref) in zip(tm.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, f"{k}: no gradient"
        worst[f"grad.{k}"] = rel_max(p.grad, p_ref.grad)
    worst["grad.x"] = rel_max(gx, gx_ref)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"{name}: worst {[(k, f'{v:.2e}') for k, v in top]}")
    assert worst.pop("out") < 1e-3
    bad = {k: v for k, v in worst.items() if v > 2.5e-4}
    assert not bad, bad
    # determinism: the same seed gives the same forward and backward, bit for bit
    grads1 = [p.grad.clone() for p in tm.parameters()] + [gx.clone()]
    out2, gx2 = native_step(tm, x, const, G, seed=17)
    assert torch.equal(out, out2)
    assert all(torch.equal(a, b) for a, b in zip(grads1, [p.grad for p in tm.parameters()] + [gx2]))


def test_sgd_step_then_eval_matches_eval_oracle():
    tm = make_model(70, 6, 3, 48, 64, 0.1).to(DEV)
    x, const = inputs(70, 6, 3, 2, 48, 64)
    x, const = x.to(DEV), const.to(DEV)
    tm.eval()
    with torch.no_grad():
        tm(x, const=const)                        # packs (and caches) the eval-mode weights
    tm.train()
    opt = torch.optim.SGD(tm.parameters(), lr=0.05)
    (tm(x, const=const) ** 2).mean().backward()
    opt.step()
    tm.eval()
    with torch.no_grad():
        got = tm(x, const=const)
        want = TD.temporal_model(full_input(x, const).double().cpu(), copy.deepcopy(tm).cpu().double())
    e = rel_max(got, want)
    assert e < 1e-3, e


def test_no_grad_train_forward_updates_running_stats():
    tm_cpu = make_model(134, 0, 5, 16, 24, 0.1)
    x, const = inputs(134, 0, 5, 1, 16, 24)
    ref = copy.deepcopy(tm_cpu).double()
    params = [p.detach().clone() for p in tm_cpu.parameters()]
    masks, keep = native_masks(tm_cpu, x, const, seed=4)
    with torch.no_grad():
        OT.temporal_model_train(x.double(), ref, dropout_mask=keep.permute(0, 3, 1, 2).cpu())
        tm = copy.deepcopy(tm_cpu).to(DEV)
        torch.manual_seed(4)
        out = tm(x.to(DEV))
    assert out.grad_fn is None
    for (k, b), (_, b_ref) in zip(tm.named_buffers(), ref.named_buffers()):
        assert rel_max(b, b_ref) < 1e-5, k
    assert all(torch.equal(p.cpu(), q) for p, q in zip(tm.parameters(), params))


@pytest.mark.parametrize("what", ["head_eval", "mixed", "bt1", "sync", "momentum_none", "standalone_block"])
def test_refusals(what):
    tm = make_model(70, 0, 3, 48, 64)
    x, _ = inputs(70, 0, 3, 2, 48, 64)
    exc, match = RuntimeError, None
    if what == "head_eval":
        tm.final_conv.eval()
        match = "final_conv is in eval mode"
    elif what == "mixed":
        tm.model[1].eval()
        match = "mixed train / eval"
    elif what == "bt1":
        x, exc, match = x[:1, :1], ValueError, "B\\*S = 1 is not supported"
    elif what == "sync":
        tm = torch.nn.SyncBatchNorm.convert_sync_batchnorm(tm)
        exc, match = NotImplementedError, "SyncBatchNorm"
    elif what == "momentum_none":
        tm.model[0].pyramid_pooling.features[0].conv_bn_relu.norm.momentum = None
        exc, match = NotImplementedError, "momentum=None"
    else:
        blk = tm.model[0].to(DEV)
        with pytest.raises(NotImplementedError, match="TemporalModel"):
            blk(x.to(DEV).permute(0, 2, 1, 3, 4))
        return
    tm = tm.to(DEV)
    with pytest.raises(exc, match=match):
        tm(x.to(DEV))


def test_autograd_node_guards():
    tm = make_model(70, 0, 3, 48, 64).to(DEV)
    x, _ = inputs(70, 0, 3, 2, 48, 64)
    x = x.to(DEV)
    loss = tm(x).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second time"):
        loss.backward()                           # the head's node refuses first
    # the blocks' own guard: drive their node directly, without the head
    params = [p for blk in tm.model for p in blk.parameters()]
    y = _TemporalBlocksTrainFn.apply(tm, x, None, *params)
    y.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match=r"TemporalModel \(train mode\): backward ran a second time"):
        y.sum().backward()
    loss = tm(x).sum()
    with torch.no_grad():
        tm.model[0].aggregation[0].conv.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()
    xg = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(tm(xg).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


# ------------------------------------------------------------------------------------------------ model level
def test_recipe_trains_everything_after_the_encoder():
    from oracle import lift_splat_oracle as O
    from stp3_b200.models.stp3 import GraphedPerception
    from stp3_b200.utils import geometry as G
    from stp3_b200.utils import synthetic as syn
    model, inp = small_stp3()
    model.train()
    model.encoder.eval()
    model.decoder.eval()
    with pytest.raises(RuntimeError, match="TemporalBlocks are in train mode"):
        GraphedPerception(model, 2, 2)
    model.decoder.train()
    feat = inp["feat"].to(DEV).requires_grad_(True)
    depth = inp["depth_logits"].to(DEV).requires_grad_(True)
    tm = model.temporal_model
    seen = {}
    hooks = [tm.register_forward_pre_hook(lambda m, a, kw: seen.update(x=a[0].detach().clone(), const=kw["const"]),
                                          with_kwargs=True),
             tm.register_forward_hook(lambda m, a, out: seen.update(y=out.detach().clone()))]
    ref_tm, ref_dec = copy.deepcopy(tm).double(), copy.deepcopy(model.decoder).double()
    tm_cpu, dec_cpu = copy.deepcopy(tm).cpu(), copy.deepcopy(model.decoder).cpu()
    before = {k: b.clone() for k, b in model.named_buffers()}
    torch.manual_seed(21)
    out = model.forward_features(feat, depth, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    for hk in hooks:
        hk.remove()
    keys = ("segmentation", "pedestrian", "hdmap")
    loss = sum(out[k].float().square().mean() for k in keys)
    loss.backward()
    for k, p in model.named_parameters():
        trained = k.startswith("temporal_model.") or k.startswith("decoder.")
        assert (p.grad is not None) == trained, k
        if trained:
            assert torch.isfinite(p.grad).all(), k
    for k, b in model.named_buffers():
        if "running" in k or "num_batches" in k:
            trained = k.startswith("temporal_model.") or k.startswith("decoder.")
            assert (not torch.equal(b, before[k])) == trained, k
    # fp64: temporal model (native ReLU branches and dropout mask pinned) -> decoder -> BEV gradient -> lift-splat bwd
    x, const = seen["x"], seen["const"]
    masks, keep = native_masks(tm_cpu, x.cpu(), const.cpu() if const is not None else None, seed=21)
    queue = list(masks)
    xd = full_input(x, const).double().requires_grad_(True)
    y = OT.temporal_model_train(xd, ref_tm.to(DEV), relu=lambda t: t * queue.pop(0),
                                dropout_mask=keep.permute(0, 3, 1, 2))
    # the decoder's ReLU branches pinned too: its input gradient is then a smooth function of the native forward
    dq = list(dec_masks(dec_cpu, seen["y"]))
    want = TT.decoder_train(y, ref_dec.to(DEV), relu=lambda t: t * dq.pop(0))
    for k in keys:
        e = rel_max(out[k].detach(), want[k].detach())
        assert e < 1e-3, (k, e)
    sum(want[k].square().mean() for k in keys).backward()
    g_bev = xd.grad[:, :, :x.shape[2]].cpu().numpy()
    lcfg = syn.LiftSplatConfig(x_bound=(-8.0, 8.0, 0.5), y_bound=(-8.0, 8.0, 0.5), d_bound=(2.0, 10.0, 1.0),
                               final_dim=(32, 48), out_channels=64, n_cameras=2, receptive_field=3)
    cam_M, cam_t, ego_R, ego_t = G.lift_matrices(inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    xs, ys, ds = G.frustum_axes(lcfg.final_dim, lcfg.downsample, lcfg.d_bound)
    res, start, dim = G.calculate_birds_eye_view_parameters(lcfg.x_bound, lcfg.y_bound, lcfg.z_bound)
    ora = O.lift_splat(inp["feat"].numpy(), inp["depth_logits"].numpy(), cam_M.numpy(), cam_t.numpy(), ego_R.numpy(),
                       ego_t.numpy(), xs.numpy(), ys.numpy(), ds.numpy(), G.bev_offset(start, res).numpy(), res.numpy(),
                       dim.numpy(), lcfg.discount)
    ogf, ogd = O.lift_splat_backward(g_bev, inp["feat"].numpy(), inp["depth_logits"].numpy(), ora["rank"], lcfg.discount)
    e_f, e_d = rel_max(feat.grad, torch.from_numpy(ogf)), rel_max(depth.grad, torch.from_numpy(ogd))
    print(f"recipe: feat.grad {e_f:.2e}, depth.grad {e_d:.2e} of max")
    assert e_f < 1e-3 and e_d < 1e-3
