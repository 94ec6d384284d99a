"""GPU: the opt-in train mode of the native EfficientNet trunk (EfficientNetTrunk(version, trainable=True).train()).

Kernel level: every new trunk entry point on synthetic shapes the trunk itself never produces (channel counts that are
not multiples of 8, one-pixel maps, odd sizes at stride 2 and k = 5, static pads that disagree with the real edge)
against fp64 models of its contract, twice bitwise.  Module level: the truncated b0 and b4
trunks at M = 4 against fp64 autograd through tests/trunk_train_reference.py with the drop-connect masks pinned
(outputs and every gradient within 1e-3 of max, running statistics within 1e-5 for b0 and 5e-5 for b4, whose deeper
layers inherit the forward's ~1e-4 error in their batch variance: DESIGN.md 3.15), one block of each kind, the bytes a
forward keeps against trunk_tape_bytes, two runs bitwise, eval mode bitwise the
default trunk's, deterministic mode, autocast and GradScaler.  Model level: a small STP3 trained from images with a
trainable b4 trunk, and the refusals."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet_oracle as EO
from stp3_b200 import dense, dense_train as T
from stp3_b200.models import efficientnet as EN
from tests import trunk_train_reference as TR

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BAR = 1e-3          # of max |fp64|: outputs and gradients (DESIGN.md 3.11's bar for the encoder heads)
RUN_BAR = {"b0": 1e-5, "b4": 5e-5}     # running statistics: b4's deeper layers inherit the forward's ~1e-4 error in
                                        # their batch variance (DESIGN.md 3.15)
WORST = {}          # name -> worst ratio, printed for DESIGN.md


def rel(got, ref):
    ref = ref.double()
    return ((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def note(name, r):
    WORST[name] = max(WORST.get(name, 0.0), r)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=gen(seed), dtype=torch.float64) * scale)


# ------------------------------------------------------------------------------------------------ kernels
def dw_model(x, w, stride, pad, Ho, Wo):
    """fp64 depthwise conv with the kernels' padding: top / left `pad`, bottom / right whatever gives Ho x Wo (negative
    crops), zeros outside.  x (N, H, W, C), w (C, 1, k, k) -> (N, Ho, Wo, C)."""
    N, H, W, C = x.shape
    k = w.shape[-1]
    pb, pr = (Ho - 1) * stride + k - H - pad, (Wo - 1) * stride + k - W - pad
    xp = F.pad(x.permute(0, 3, 1, 2), (pad, pr, pad, pb))
    return F.conv2d(xp, w, stride=stride, groups=C).permute(0, 2, 3, 1)


DW_CASES = [  # N, H, W, C, k, s, pad, Ho, Wo
    (2, 9, 11, 24, 5, 2, 1, 5, 6),      # b4-like static pad (1, 2) on an odd map: the real edge disagrees
    (2, 9, 11, 24, 5, 2, 2, 5, 6),
    (3, 7, 7, 12, 3, 2, 0, 4, 4),       # pad (0, 1) at the nominal size, C not a multiple of 8
    (1, 1, 1, 70, 3, 1, 1, 1, 1),       # one pixel
    (1, 1, 1, 5, 5, 2, 1, 1, 1),
    (2, 13, 6, 1, 5, 1, 2, 13, 6),
    (2, 10, 14, 40, 3, 1, 1, 10, 14),
    (1, 28, 60, 136, 5, 2, 1, 14, 30),  # a wide stride-2 5x5 layer on an even map
]


@pytest.mark.parametrize("case", DW_CASES)
def test_depthwise_kernels_against_fp64(case):
    N, H, W, C, k, s, pad, Ho, Wo = case
    x64 = randn((N, H, W, C), 1).requires_grad_(True)
    w64 = randn((C, 1, k, k), 2, 0.3).requires_grad_(True)
    g64 = randn((N, Ho, Wo, C), 3)
    y64 = dw_model(x64, w64, s, pad, Ho, Wo)
    y64.backward(g64)
    x, w, g = (t.detach().float().to(DEV).contiguous() for t in (x64, w64, g64))
    outs = []
    for _ in range(2):
        y = T.dw_raw(x, w, s, pad, (Ho, Wo))
        dx = T.dw_dgrad(g, w, s, pad, (H, W))
        dw = T.dw_wgrad(x, g, k, s, pad)
        outs.append((y, dx, dw))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    y, dx, dw = outs[0]
    assert rel(y.cpu(), y64.detach()) < 1e-6, rel(y.cpu(), y64.detach())
    assert rel(dx.cpu(), x64.grad) < 1e-6, rel(dx.cpu(), x64.grad)
    # the weight gradient adds in fp64 and rounds once: the exact sum of the fp32 operands, to one fp32 rounding
    wr = w64.detach().clone().requires_grad_(True)
    exact, = torch.autograd.grad(dw_model(x.double().cpu(), wr, s, pad, Ho, Wo), [wr], g.double().cpu())
    mag, = torch.autograd.grad(dw_model(x.double().cpu().abs(), wr, s, pad, Ho, Wo), [wr], g.double().cpu().abs())
    assert ((dw.double().cpu() - exact).abs() <= 2 ** -24 * exact.abs() + 1e-13 * mag).all()


def test_stem_kernels_against_fp64():
    for (M, H, W, cout, pad) in ((2, 17, 23, 48, 1), (1, 1, 1, 5, 0), (3, 12, 9, 32, 0), (1, 6, 8, 64, 1)):
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        x64 = randn((M, 3, H, W), 4)
        w64 = randn((cout, 3, 3, 3), 5, 0.3).requires_grad_(True)
        pb, pr = (Ho - 1) * 2 + 3 - H - pad, (Wo - 1) * 2 + 3 - W - pad
        y64 = F.conv2d(F.pad(x64, (pad, pr, pad, pb)), w64, stride=2).permute(0, 2, 3, 1)
        g64 = randn(y64.shape, 6)
        y64.backward(g64)
        x, w, g = (t.detach().float().to(DEV).contiguous() for t in (x64, w64, g64))
        y = T.stem_raw(x, w, (Ho, Wo), pad)
        dw = T.stem_wgrad(x, g.contiguous(), pad)
        assert torch.equal(dw, T.stem_wgrad(x, g.contiguous(), pad))
        assert rel(y.cpu(), y64.detach()) < 1e-6
        wr = w64.detach().clone().requires_grad_(True)
        xf, gf = x.double().cpu(), g.double().cpu()
        exact, = torch.autograd.grad(F.conv2d(F.pad(xf, (pad, pr, pad, pb)), wr, stride=2).permute(0, 2, 3, 1), [wr], gf)
        mag, = torch.autograd.grad(F.conv2d(F.pad(xf.abs(), (pad, pr, pad, pb)), wr, stride=2).permute(0, 2, 3, 1), [wr],
                                   gf.abs())
        assert ((dw.double().cpu() - exact).abs() <= 2 ** -24 * exact.abs() + 1e-13 * mag).all()


def _stats(x):
    return T.bn_stats(x, 1e-3, 0.1)


@pytest.mark.parametrize("C,hl", [(24, True), (13, True), (70, False), (1, True)])
def test_bn_act_and_its_gradient_against_fp64(C, hl):
    N, H, W = 3, 5, 7
    x = randn((N, H, W, C), 7).float().to(DEV)
    bn = torch.nn.BatchNorm2d(C, eps=1e-3).to(DEV)
    with torch.no_grad():
        bn.weight.copy_(randn((C,), 8).abs().float() + 0.5)
        bn.bias.copy_(randn((C,), 9, 0.1).float())
    st = _stats(x)
    mul = torch.rand((N, C), generator=gen(1)).to(DEV)
    add = randn((N, C), 10, 0.01).float().to(DEV)
    scale = torch.tensor([0.0, 1.25, 1.25])[:N].to(DEV)
    res = randn((N, H, W, C), 11).float().to(DEV)
    z64 = (x.double() - st.mean.double()) * st.invstd.double() * bn.weight.double() + bn.bias.double()
    for swish in (True, False):
        a64 = z64 * torch.sigmoid(z64) if swish else z64
        y, planes = T.bn_act(x, st, bn, swish, mul=mul, scale=scale, res=res, hl=hl)
        ref = a64 * mul.double().view(N, 1, 1, C) * scale.double().view(N, 1, 1, 1) + res.double()
        assert rel(y, ref) < 1e-6
        if hl:
            assert planes.hi.shape[-1] == dense.pad_to(C)
            back = (planes.hi.float() + planes.lo.float())[..., :C].reshape(y.shape)
            assert rel(back, y.double()) < 2 ** -16
            assert (planes.hi[..., C:] == 0).all() and (planes.lo[..., C:] == 0).all()
        g = randn((N, H, W, C), 12).float().to(DEV)
        out = T.bn_act_grad(g, x, st, bn, swish, mul=mul, add=add, scale=scale)
        s = torch.sigmoid(z64)
        d = s * (1 + z64 * (1 - s)) if swish else torch.ones_like(z64)
        ref = (g.double() * mul.double().view(N, 1, 1, C) + add.double().view(N, 1, 1, C)) * d * \
            scale.double().view(N, 1, 1, 1)
        assert rel(out, ref) < 1e-6
        assert torch.equal(out, T.bn_act_grad(g, x, st, bn, swish, mul=mul, add=add, scale=scale))
    # no statistics: the gate alone
    y, _ = T.bn_act(x, None, None, False, mul=mul)
    assert rel(y, x.double() * mul.double().view(N, 1, 1, C)) < 1e-7


@pytest.mark.parametrize("N,H,W,C", [(3, 5, 7, 24), (2, 1, 1, 13), (1, 30, 41, 96), (2, 60, 120, 8)])
def test_image_channel_dot_against_fp64(N, H, W, C):
    a, b = randn((N, H, W, C), 13).float().to(DEV), randn((N, H, W, C), 14).float().to(DEV)
    got = T.image_channel_dot(a, b)
    ref = (a.double() * b.double()).sum(dim=(1, 2))
    mag = (a.double() * b.double()).abs().sum(dim=(1, 2))
    assert ((got.double() - ref).abs() <= 2 ** -24 * ref.abs() + 1e-12 * mag).all()
    assert torch.equal(got, T.image_channel_dot(a, b))


@pytest.mark.parametrize("N,C,R,hw", [(4, 96, 4, 35), (2, 13, 1, 1), (3, 960, 40, 28)])
def test_se_backward_against_fp64(N, C, R, hw):
    sums = randn((N, C), 15, hw).float().to(DEV)
    w_r = randn((R, C), 16, C ** -0.5).float().to(DEV)
    b_r = randn((R,), 17, 0.1).float().to(DEV)
    w_e = randn((C, R), 18, R ** -0.5).float().to(DEV)
    b_e = randn((C,), 19, 0.1).float().to(DEV)
    gate = torch.empty((N, C), device=DEV)
    dense.se_gate(sums, hw, C, w_r, b_r, w_e, b_e, torch.zeros((1, C), device=DEV), gate=gate)
    dgate = randn((N, C), 20).float().to(DEV)
    de, sr, dr, dmean = T.se_backward(dgate, gate, sums, hw, w_r, b_r, w_e)
    m = (sums.double() / hw).requires_grad_(True)
    W_r, B_r, W_e, B_e = (t.double().requires_grad_(True) for t in (w_r, b_r, w_e, b_e))
    r = m @ W_r.t() + B_r
    srr = r * torch.sigmoid(r)
    e = srr @ W_e.t() + B_e
    gt = torch.sigmoid(e)
    assert rel(gate, gt.detach()) < 1e-6
    gt.backward(dgate.double())
    assert rel(sr, srr.detach()) < 1e-6
    assert rel(de.sum(0), B_e.grad) < 1e-5 and rel(dr.sum(0), B_r.grad) < 1e-5
    assert rel(dmean * hw, m.grad) < 1e-5
    assert rel(T.conv_wgrad(sr.view(N, 1, 1, R), de.view(N, 1, 1, C), 1, 1, 1).view(C, R), W_e.grad) < 1e-5
    assert rel(T.conv_wgrad((sums / hw).view(N, 1, 1, C), dr.view(N, 1, 1, R), 1, 1, 1).view(R, C), W_r.grad) < 1e-5


# ------------------------------------------------------------------------------------------------ modules
def pair(version, seed=3, momentum=0.1):
    """(native trainable trunk on the GPU, fp64 restatement on the CPU), same weights and running statistics"""
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=seed), version)
    for m in ora.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = momentum
    nat = EN.EfficientNetTrunk(version, trainable=True)
    nat.load_state_dict(ora.state_dict(), strict=True)
    for m in nat.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = momentum
    return nat.to(DEV), ora.double()


def images(M, H, W, seed=21):
    return randn((M, 3, H, W), seed).float()


def zero_grad_params(trunk):
    """Parameters whose exact gradient is zero: _bn2.bias of a block whose output (followed along the identity skips of
    the blocks after it) reaches neither endpoint and only feeds 1x1 expand convolutions into batch-statistics _bn0
    layers, which remove a per-channel constant.  Their fp32 gradient is rounding noise, so it is held to the bar
    relative to the same BatchNorm's weight gradient."""
    out = {}
    n = len(trunk._blocks)
    for i in range(n):
        j = i
        while j + 1 < n and trunk._blocks[j + 1].spec.skip:
            j += 1
        if j not in (trunk.endpoint, n - 1) and all(trunk._blocks[b].spec.exp != trunk._blocks[b].spec.cin
                                                    for b in range(i + 1, j + 2)):
            out[f"_blocks.{i}._bn2.bias"] = f"_blocks.{i}._bn2.weight"
    return out


def check_grads(nat, ora, name, zero=None):
    po = dict(ora.named_parameters())
    zero = zero_grad_params(nat) if zero is None else zero
    bad, worst = [], 0.0
    for k, p in nat.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        ref = po[k].grad
        if k in zero:
            r = ((p.grad.cpu().double() - ref).abs().max() / po[zero[k]].grad.abs().max()).item()
        else:
            r = rel(p.grad.cpu(), ref)
        worst = max(worst, r)
        if not r < BAR:
            bad.append((k, r))
    note(f"{name} gradients", worst)
    assert not bad, bad


def run_native(nat, x, seed, g3, g4):
    torch.manual_seed(seed)
    nat.train()
    r3, r4 = nat(x.to(DEV))
    (r3 * g3.to(DEV)).sum().add((r4 * g4.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    return r3.detach(), r4.detach()


def run_reference(ora, x, masks, g3, g4):
    ora.train()
    r3, r4 = TR.trunk_forward(ora, x.double(), {k: v.double().cpu() for k, v in masks.items()})
    (r3 * g3.double()).sum().add((r4 * g4.double()).sum()).backward()
    return r3.detach(), r4.detach()


@pytest.mark.parametrize("version,M,H,W", [("b0", 4, 64, 96), ("b4", 4, 64, 96), ("b4", 4, 35, 51)])
def test_trunk_train_step_against_fp64(version, M, H, W):
    nat, ora = pair(version)
    x = images(M, H, W)
    torch.manual_seed(5)
    masks = TR.draw_masks(ora, M, DEV)
    with torch.no_grad():
        r3s, r4s = TR.trunk_forward(copy.deepcopy(ora).eval(), x.double())
    g3, g4 = randn(r3s.shape, 31), randn(r4s.shape, 32)
    got3, got4 = run_native(nat, x, 5, g3, g4)
    ref3, ref4 = run_reference(ora, x, masks, g3, g4)
    note(f"{version} outputs", max(rel(got3.cpu(), ref3), rel(got4.cpu(), ref4)))
    print(version, "outputs", rel(got3.cpu(), ref3), rel(got4.cpu(), ref4))
    assert rel(got3.cpu(), ref3) < BAR and rel(got4.cpu(), ref4) < BAR
    check_grads(nat, ora, version)
    bo = dict(ora.named_buffers())
    for k, b in nat.named_buffers():
        if k.endswith("num_batches_tracked"):
            assert int(b) == 1, k
        else:
            r = rel(b.cpu(), bo[k])
            note(f"{version} running statistics", r)
            assert r < RUN_BAR[version], (k, r)
    print("worst ratios:", WORST)


@pytest.mark.parametrize("i,kind", [(0, "no expand"), (2, "expand + stride 2"), (3, "skip with drop-connect")])
def test_one_block_of_each_kind_against_fp64(i, kind):
    nat, ora = pair("b4")
    blk, oblk = nat._blocks[i], ora._blocks[i]
    s = blk.spec
    assert (s.exp == s.cin) == (kind == "no expand") and (s.stride == 2) == (kind == "expand + stride 2")
    assert s.skip == (kind == "skip with drop-connect")
    M, H, W = 4, 13, 18
    rate = EN.drop_connect_rates(len(nat._blocks))[i]
    mask = torch.tensor([1.0, 0.0, 1.0, 1.0])
    scale = (mask / (1.0 - rate)).to(DEV) if s.skip else None
    xin = randn((M, H, W, s.cin), 40).float().to(DEV)
    out, _, tape = nat._train_block(blk, xin, T.to_hl(xin) if s.exp != s.cin else None, scale, False)
    g = randn(out.shape, 41).float().to(DEV)
    grads = {}
    dx = nat._block_backward(blk, tape, g, grads)
    x64 = xin.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
    oblk.train()
    y64 = TR.block_forward(oblk, x64, rate, mask.double() if s.skip else None)
    y64.backward(g.double().cpu().permute(0, 3, 1, 2))
    assert rel(out.cpu().permute(0, 3, 1, 2), y64.detach()) < BAR
    assert rel(dx.cpu().permute(0, 3, 1, 2), x64.grad) < BAR
    po = dict(oblk.named_parameters())
    for k, p in blk.named_parameters():
        r = rel(grads[p].cpu(), po[k].grad)
        note(f"block {i} ({kind}) gradients", r)
        assert r < BAR, (k, r)
    bo = dict(oblk.named_buffers())
    for k, b in blk.named_buffers():
        if not k.endswith("num_batches_tracked"):
            assert rel(b.cpu(), bo[k]) < RUN_BAR["b0"], k


@pytest.mark.parametrize("version", ["b0", "b4"])
def test_forward_keeps_the_tape_the_formula_counts(version):
    nat, _ = pair(version)
    M, H, W = 3, 64, 96
    x = images(M, H, W).to(DEV)
    nat.train()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    r3, r4 = nat(x)
    torch.cuda.synchronize()
    kept = torch.cuda.memory_allocated() - before
    tape = M * EN.trunk_tape_bytes(version, H, W)
    # beyond the activations: per-channel statistics, gates, sums and the allocator's 512-byte rounding
    assert tape <= kept <= 1.05 * tape, (kept, tape)
    (r3.sum() + r4.sum()).backward()


def test_two_runs_bitwise_and_eval_matches_the_default_trunk():
    nat, ora = pair("b4")
    x = images(4, 64, 96)
    g3, g4 = randn((4, 56, 8, 12), 33), randn((4, 160, 4, 6), 34)
    res = []
    for _ in range(2):
        n = copy.deepcopy(nat)
        out = run_native(n, x, 9, g3, g4)
        res.append((out, [p.grad.clone() for p in n.parameters()], [b.clone() for b in n.buffers()]))
    (a3, a4), ga, ba = res[0]
    (b3, b4), gb, bb = res[1]
    assert torch.equal(a3, b3) and torch.equal(a4, b4)
    assert all(torch.equal(u, v) for u, v in zip(ga, gb)) and all(torch.equal(u, v) for u, v in zip(ba, bb))
    # eval mode of the trainable trunk is the default trunk, bit for bit (timing-free convolution tilings, so the two
    # packings run the same tiling)
    default = EN.EfficientNetTrunk("b4").to(DEV)
    default.load_state_dict(nat.state_dict())
    nat.eval()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            e1, e2 = nat(x.to(DEV)), default(x.to(DEV))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(e1[0], e2[0]) and torch.equal(e1[1], e2[1])


def test_deterministic_mode_two_steps_bitwise():
    nat, _ = pair("b0")
    x = images(3, 48, 64)
    g3, g4 = randn((3, 40, 6, 8), 35), randn((3, 112, 3, 4), 36)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        res = []
        for _ in range(2):
            n = copy.deepcopy(nat)
            out = run_native(n, x, 13, g3, g4)
            res.append((out, [p.grad.clone() for p in n.parameters()], [b.clone() for b in n.buffers()]))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(u, v) for u, v in zip(res[0][0], res[1][0]))
    assert all(torch.equal(u, v) for u, v in zip(res[0][1], res[1][1]))
    assert all(torch.equal(u, v) for u, v in zip(res[0][2], res[1][2]))


def test_autocast_is_ignored_and_gradscaler_skips_an_overflowed_step():
    nat, _ = pair("b0")
    x = images(2, 48, 64).to(DEV)
    a = copy.deepcopy(nat).train()
    torch.manual_seed(3)
    f32 = a(x)
    b = copy.deepcopy(nat).train()
    torch.manual_seed(3)
    with torch.autocast("cuda", dtype=torch.float16):
        amp = b(x)
    assert amp[0].dtype == torch.float32 and torch.equal(f32[0], amp[0]) and torch.equal(f32[1], amp[1])
    # GradScaler: a scale that overflows the loss gives non-finite gradients, the step is skipped, the next one runs
    n = copy.deepcopy(nat).train()
    opt = torch.optim.Adam(n.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 126)
    before = [p.detach().clone() for p in n.parameters()]
    for step in range(2):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            r3, r4 = n(x)
            loss = r3.float().square().mean() + r4.float().square().mean() * 1e6
        scaler.scale(loss).backward()
        scaler.step(opt)
        if step == 0:
            assert all(torch.equal(p, q) for p, q in zip(n.parameters(), before)), "overflowed step was not skipped"
        scaler.update(1.0 if step == 0 else None)
    assert all(torch.isfinite(p).all() for p in n.parameters())
    assert any(not torch.equal(p, q) for p, q in zip(n.parameters(), before))


def test_autograd_guards():
    nat, _ = pair("b0")
    x = images(2, 48, 64).to(DEV)
    nat.train()
    r3, r4 = nat(x)
    loss = r3.sum() + r4.sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="backward ran a second time"):
        loss.backward()
    r3, r4 = nat(x)
    with torch.no_grad():
        nat._blocks[1]._depthwise_conv.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        (r3.sum() + r4.sum()).backward()


# ------------------------------------------------------------------------------------------------ model
def test_stp3_trains_every_parameter_from_images():
    from tests.test_encoder_train_gpu import LCFG, gauss, loss_of, small_stp3
    from stp3_b200.models.stp3 import GraphedPerception
    model, inp = small_stp3(EN.EfficientNetTrunk("b4", trainable=True))
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle("b4"), seed=5), "b4")
    model.encoder.backbone.load_state_dict(ora.state_dict(), strict=True)
    for m in ora.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = model.encoder.backbone._bn0.momentum
    model = model.to(DEV).train()
    image = gauss((1, 3, 2, 3, *LCFG.final_dim), 3).to(DEV)
    # refusals
    with pytest.raises(NotImplementedError, match="images is not computed"):
        model(image.clone().requires_grad_(True), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    model.encoder.train_heads(False)
    with pytest.raises(RuntimeError, match="native trunk is in train mode but the encoder heads are in eval mode"):
        model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    model.eval()
    model.encoder.backbone.train()
    for entry in ("images", "lift"):
        with pytest.raises(RuntimeError, match="native trunk is in train mode"):
            GraphedPerception(model, 1, 2, entry=entry)
    with pytest.raises(RuntimeError, match="native trunk is in train mode"):
        model.forward_features_frame_sharded(inp["feat"].to(DEV), inp["depth_logits"].to(DEV), inp["intrinsics"],
                                             inp["extrinsics"], inp["future_egomotion"])
    # a graph captured before the step (eval mode) must refuse to replay once the step has changed the weights
    model.eval()
    graphed = GraphedPerception(model, 1, 2, entry="images")
    model.train()
    # one train step; capture the endpoint gradients to drive the fp64 trunk
    trunk = model.encoder.backbone
    cap = {}
    fwd = trunk.forward_train

    def capture(x):
        torch.manual_seed(17)
        r3, r4 = fwd(x)
        cap["x"] = x.detach().cpu()
        r3.retain_grad()
        r4.retain_grad()
        cap["r"] = (r3, r4)
        return r3, r4
    trunk.forward_train = capture
    try:
        out = model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        loss_of(out).backward()
    finally:
        del trunk.forward_train
    torch.cuda.synchronize()
    for k, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
            if k.startswith("encoder.backbone."):
                assert p.grad.abs().max() > 0, k
    for k, b in model.named_buffers():
        if k.endswith("num_batches_tracked") and k.startswith("encoder.backbone."):
            assert int(b) == 1, k
    torch.manual_seed(17)
    M = cap["x"].shape[0]
    masks = TR.draw_masks(ora, M, DEV)
    ora = ora.double().train()
    g3, g4 = (r.grad.detach().cpu().double() for r in cap["r"])
    run_reference(ora, cap["x"], masks, g3, g4)
    # behind the heads every endpoint feeds batch-statistics BatchNorms, which remove per-channel constants: every
    # _bn2.bias gradient is near zero (only the heads' zero padding leaves a trace), held relative to its _bn2.weight's
    check_grads(trunk, ora, "STP3 b4 trunk", {f"_blocks.{i}._bn2.bias": f"_blocks.{i}._bn2.weight"
                                              for i in range(len(trunk._blocks))})
    print("worst ratios:", WORST)
    # an optimizer step, then the eval forward repacks the trunk from the new weights
    model.eval()
    with torch.no_grad():
        e0 = trunk(image.view(-1, *image.shape[3:]))
    torch.optim.Adam(model.parameters(), lr=1e-3).step()
    with torch.no_grad():
        e1 = trunk(image.view(-1, *image.shape[3:]))
    assert not torch.equal(e0[1], e1[1])
    with pytest.raises(RuntimeError, match="parameters changed after the CUDA graph was captured"):
        graphed(image, None, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
    ref = EN.EfficientNetTrunk("b4").to(DEV)
    ref.load_state_dict(trunk.state_dict())
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            e1 = trunk(image.view(-1, *image.shape[3:]))
            e2 = ref(image.view(-1, *image.shape[3:]))
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(e1[1], e2[1])
