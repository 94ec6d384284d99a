"""GPU: the train-mode modules under torch.autocast (float16 and bfloat16), against the fp64 oracles and against torch's
own AMP.

Each module runs one step with the forward under autocast and the backward outside it (as Lightning runs a
precision=16 step).  Its error against fp64 autograd through the train-mode restatement (oracle/torch_*_train.py, ReLU
branches and dropout masks pinned to the native forward's) must stay within twice the error of the same restatement
run in fp32 under the same autocast region -- torch's AMP on the same inputs -- plus a small floor, for the outputs,
every parameter gradient and the input gradients; running statistics must be updated.  Loss scaling: GradScaler skips a
step whose gradients overflowed and otherwise returns the unscaled step's gradients (DeepLab head); whole STP3 models
behind a torch trunk (model.train()) and behind the native trunk (the train_heads() recipe) skip an overflowed step
and train stably with GradScaler and Adam; and the precision mode follows the forward, not the backward's autocast
state."""
import copy

import pytest
import torch

from oracle import torch_deeplab_train as OD
from oracle import torch_dense_train as OT
from oracle import torch_encoder_train as OE
from oracle import torch_temporal_train as OTT
from stp3_b200.layers.convolutions import UpsamplingConcat
from tests import test_decoder_train_gpu as TDEC
from tests import test_deeplab_train_gpu as TDL
from tests import test_temporal_train_gpu as TTM

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODES = [torch.float16, torch.bfloat16]
FLOOR = 1e-4
# the one-product path is in use: the native outputs' error is of torch-AMP's size, not the ~1e-6 of the hi/lo path
ENGAGED = 0.25
gauss, rel_max = TDL.gauss, TDL.rel_max


def pinned(masks):
    queue = list(masks)
    return queue, (lambda t: t * queue.pop(0).to(t.device, t.dtype))


def compare(name, mode, native, ref64, amp, skip=()):
    """native / ref64 / amp: (outputs dict, module, input gradients dict) -> asserts the 2x-of-torch-AMP bar"""
    (o_n, m_n, gx_n), (o_r, m_r, gx_r), (o_a, m_a, gx_a) = native, ref64, amp
    errs = {}
    for k in o_r:
        errs[f"out.{k}"] = (rel_max(o_n[k].detach(), o_r[k].detach()), rel_max(o_a[k].detach(), o_r[k].detach()))
    for (k, p), (_, pr), (_, pa) in zip(m_n.named_parameters(), m_r.named_parameters(), m_a.named_parameters()):
        if k in skip:
            continue
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
        errs[f"grad.{k}"] = (rel_max(p.grad, pr.grad), rel_max(pa.grad, pr.grad))
    for k in gx_r:
        errs[f"grad.{k}"] = (rel_max(gx_n[k], gx_r[k]), rel_max(gx_a[k], gx_r[k]))
    for (k, b), (_, br) in zip(m_n.named_buffers(), m_r.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert int(b) == int(br) == 1, k
        else:
            assert rel_max(b, br) < 2e-2, (k, rel_max(b, br))
    outs = [v for k, v in errs.items() if k.startswith("out.")]
    assert max(n for n, _ in outs) >= ENGAGED * max(a for _, a in outs), ("still on the fp32-equivalent path?", outs)
    worst = sorted(errs.items(), key=lambda kv: -kv[1][0] / (2 * kv[1][1] + FLOOR))[:3]
    print(f"{name} {mode}: worst native / torch-AMP errors {[(k, f'{a:.1e}/{b:.1e}') for k, (a, b) in worst]}")
    bad = {k: v for k, v in errs.items() if v[0] > 2 * v[1] + FLOOR}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ DeepLabHead
def deeplab_native(head, x, G, seed, mode, backward_in_autocast=False):
    xx = x.to(DEV).requires_grad_(True)
    head.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    with torch.autocast("cuda", dtype=mode, enabled=mode is not None):
        out = head(xx)
        if backward_in_autocast:
            (out * G.to(DEV)).sum().backward()
    if not backward_in_autocast:
        (out * G.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    return out, xx.grad


def deeplab_oracle(head_cpu, x, G, masks, keep, mode):
    ref = copy.deepcopy(head_cpu).to(DEV)
    ref = ref.double() if mode is None else ref
    xd = x.to(DEV, torch.float64 if mode is None else torch.float32).requires_grad_(True)
    queue, relu = pinned(masks)
    with torch.autocast("cuda", dtype=mode or torch.float16, enabled=mode is not None):
        out = OD.deeplab_head_train(xd, ref, relu=relu, dropout_mask=keep.permute(0, 3, 1, 2))
    assert not queue
    (out.to(xd.dtype) * G.to(DEV, xd.dtype)).sum().backward()
    return out, ref, xd.grad


@pytest.mark.parametrize("mode", MODES)
def test_deeplab_head_under_autocast(mode):
    cin, ncls, hidden, N, H, W = 64, 64, 128, 6, 48, 64
    head_cpu = TDL.make_head(cin, ncls, hidden)
    x = gauss((N, cin, H, W), 5)
    G = gauss((N, ncls, H, W), 9) * 0.25
    with torch.autocast("cuda", dtype=mode):
        masks, keep = TDL.native_masks(head_cpu, x, seed=17)
    head = copy.deepcopy(head_cpu).to(DEV)
    out, gx = deeplab_native(head, x, G, 17, mode)
    assert out.dtype == torch.float32
    o64, r64, gx64 = deeplab_oracle(head_cpu, x, G, masks, keep, None)
    oa, ra, gxa = deeplab_oracle(head_cpu, x, G, masks, keep, mode)
    compare("DeepLabHead", mode, ({"y": out}, head, {"x": gx}), ({"y": o64}, r64, {"x": gx64}), ({"y": oa}, ra, {"x": gxa}))


# ------------------------------------------------------------------------------------------------ UpsamplingConcat
def upcat_masks(mod_cpu, x_up, x, mode):
    mod = copy.deepcopy(mod_cpu).to(DEV)
    with torch.no_grad(), torch.autocast("cuda", dtype=mode):
        _, tape = mod._train_forward(x_up.to(DEV), x.to(DEV), False)
    return [(tape[k] > 0).permute(0, 3, 1, 2).double() for k in ("y0", "y1")]


@pytest.mark.parametrize("mode", MODES)
def test_upsampling_concat_under_autocast(mode):
    mod_cpu = TDL.TD.init_exact(UpsamplingConcat(64 + 128, 64), seed=4).train()
    x_up, x = gauss((4, 128, 14, 30), 6), gauss((4, 64, 28, 60), 7)
    G = gauss((4, 64, 28, 60), 8) * 0.25
    x_up, x = x_up.to(mode).float(), x.to(mode).float()        # the 16-bit inputs an autocast region hands over
    masks = upcat_masks(mod_cpu, x_up, x, mode)
    mod = copy.deepcopy(mod_cpu).to(DEV)
    # fp16 inputs from an autocast region are accepted; their gradients come back in fp16
    xu = x_up.to(DEV, mode).requires_grad_(True)
    xx = x.to(DEV, mode).requires_grad_(True)
    with torch.autocast("cuda", dtype=mode):
        out = mod(xu, xx)
    (out * G.to(DEV)).sum().backward()
    assert out.dtype == torch.float32 and xu.grad.dtype == mode and xx.grad.dtype == mode
    runs = []
    for m in (None, mode):
        ref = copy.deepcopy(mod_cpu).to(DEV)
        dt = torch.float64 if m is None else torch.float32
        ref = ref.to(dt)
        a = x_up.to(DEV, mode).to(dt).requires_grad_(True)
        b = x.to(DEV, mode).to(dt).requires_grad_(True)
        queue, relu = pinned(masks)
        with torch.autocast("cuda", dtype=m or torch.float16, enabled=m is not None):
            o = OE.upsampling_concat_train(a, b, ref, relu=relu)
        (o.to(dt) * G.to(DEV, dt)).sum().backward()
        runs.append(({"y": o}, ref, {"x_up": a.grad, "x": b.grad}))
    compare("UpsamplingConcat", mode, ({"y": out}, mod, {"x_up": xu.grad, "x": xx.grad}), *runs)


# ------------------------------------------------------------------------------------------------ Decoder
@pytest.mark.parametrize("mode", MODES)
def test_decoder_under_autocast(mode):
    dec_cpu = TDEC.make_decoder(TDEC.GATES_PERCEIVE)
    x = gauss((2, 3, 64, 48, 64), 1)
    with torch.autocast("cuda", dtype=mode):
        masks = TDEC.native_relu_masks(dec_cpu, x)
    dec = copy.deepcopy(dec_cpu).to(DEV)
    xx = x.to(DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=mode):
        out = dec(xx)
    G = {k: gauss(tuple(v.shape), 10 + i) * 0.25 for i, (k, v) in enumerate(out.items()) if v is not None}
    sum((out[k] * G[k].to(DEV)).sum() for k in G).backward()
    runs = []
    for m in (None, mode):
        dt = torch.float64 if m is None else torch.float32
        ref = copy.deepcopy(dec_cpu).to(DEV).to(dt)
        xd = x.to(DEV, dt).requires_grad_(True)
        queue, relu = pinned(masks)
        with torch.autocast("cuda", dtype=m or torch.float16, enabled=m is not None):
            o = OT.decoder_train(xd, ref, relu=relu)
        sum((o[k].to(dt) * G[k].to(DEV, dt)).sum() for k in G).backward()
        runs.append(({k: o[k] for k in G}, ref, {"x": xd.grad}))
    compare("Decoder", mode, ({k: out[k] for k in G}, dec, {"x": xx.grad}), *runs, skip=TDEC.ZERO_GRAD)


# ------------------------------------------------------------------------------------------------ TemporalModel
@pytest.mark.parametrize("mode", MODES)
def test_temporal_model_under_autocast(mode):
    cin, nc, S, B, H, W = 70, 6, 3, 2, 48, 64
    tm_cpu = TTM.make_model(cin, nc, S, H, W)
    x, const = TTM.inputs(cin, nc, S, B, H, W)
    G = gauss((B, S, 64, H, W), 9) * 0.25
    with torch.autocast("cuda", dtype=mode):
        masks, keep = TTM.native_masks(tm_cpu, x, const, seed=17)
    tm = copy.deepcopy(tm_cpu).to(DEV)
    xx = x.to(DEV).requires_grad_(True)
    torch.manual_seed(17)
    with torch.autocast("cuda", dtype=mode):
        out = tm(xx, const=const.to(DEV))
    (out * G.to(DEV)).sum().backward()
    runs = []
    for m in (None, mode):
        dt = torch.float64 if m is None else torch.float32
        ref = copy.deepcopy(tm_cpu).to(DEV).to(dt)
        xd = TTM.full_input(x, const).to(DEV, dt).requires_grad_(True)
        queue, relu = pinned(masks)
        with torch.autocast("cuda", dtype=m or torch.float16, enabled=m is not None):
            o = OTT.temporal_model_train(xd, ref, relu=relu, dropout_mask=keep.permute(0, 3, 1, 2))
        (o.to(dt) * G.to(DEV, dt)).sum().backward()
        runs.append(({"y": o}, ref, {"x": xd.grad[:, :, :x.shape[2]]}))
    compare("TemporalModel", mode, ({"y": out}, tm, {"x": xx.grad}), *runs)


# ------------------------------------------------------------------------------------------------ loss scaling
def test_grad_scaler_skips_overflow_and_unscales():
    cin, ncls, hidden, N, H, W = 64, 64, 128, 4, 32, 48
    head_cpu = TDL.make_head(cin, ncls, hidden)
    x = gauss((N, cin, H, W), 5).to(DEV)
    G = (gauss((N, ncls, H, W), 9) * 0.25).to(DEV)

    def step(head, scaler, opt=None):
        head.zero_grad(set_to_none=True)
        torch.manual_seed(3)
        with torch.autocast("cuda", dtype=torch.float16):
            loss = (head(x) * G).sum()
        if scaler is None:
            loss.backward()
            return None
        scaler.scale(loss).backward()
        if opt is not None:
            scaler.step(opt)
            scaler.update()
        return scaler

    # an overflowing scale: the gradients carry inf / NaN, the step is skipped and the scale drops
    head = copy.deepcopy(head_cpu).to(DEV)
    before = [p.detach().clone() for p in head.parameters()]
    opt = torch.optim.Adam(head.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    step(head, scaler, opt)
    assert scaler.get_scale() < 2.0 ** 40
    assert all(torch.equal(a, b) for a, b in zip(before, head.parameters()))
    # a moderate scale: unscaled gradients equal the unscaled step's
    ref = copy.deepcopy(head_cpu).to(DEV)
    step(ref, None)
    scaled = copy.deepcopy(head_cpu).to(DEV)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 8)
    step(scaled, scaler)
    for (k, p), (_, pr) in zip(scaled.named_parameters(), ref.named_parameters()):
        e = rel_max(p.grad / 2.0 ** 8, pr.grad)
        assert e < 1e-2, (k, e)
    # a few Adam steps stay finite
    head = copy.deepcopy(head_cpu).to(DEV)
    opt = torch.optim.Adam(head.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    for _ in range(4):
        step(head, scaler, opt)
    assert all(bool(torch.isfinite(p).all()) for p in head.parameters())


# ------------------------------------------------------------------------------------------------ mode follows the forward
def test_mode_is_taken_from_the_forward():
    cin, ncls, hidden, N, H, W = 64, 64, 128, 4, 32, 48
    head_cpu = TDL.make_head(cin, ncls, hidden)
    x, G = gauss((N, cin, H, W), 5), gauss((N, ncls, H, W), 9)

    def grads(mode, bwd_in):
        head = copy.deepcopy(head_cpu).to(DEV)
        out, gx = deeplab_native(head, x, G, 17, mode, backward_in_autocast=bwd_in)
        return [out.detach()] + [p.grad for p in head.parameters()] + [gx]

    # forward under fp16 autocast: the backward uses the recorded one-product mode wherever it runs
    a, b = grads(torch.float16, False), grads(torch.float16, True)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    # forward outside autocast: bit for bit the fp32 path, even with the backward inside an autocast region
    plain = grads(None, False)
    head = copy.deepcopy(head_cpu).to(DEV)
    xx = x.to(DEV).requires_grad_(True)
    torch.manual_seed(17)
    out = head(xx)
    with torch.autocast("cuda", dtype=torch.float16):
        (out * G.to(DEV)).sum().backward()
    mixed = [out.detach()] + [p.grad for p in head.parameters()] + [xx.grad]
    assert all(torch.equal(u, v) for u, v in zip(plain, mixed))
    assert not all(torch.equal(u, v) for u, v in zip(plain, a))


# ------------------------------------------------------------------------------------------------ whole model
def _model_scaler_checks(make, image, inp, trained):
    """GradScaler + Adam on a train-mode STP3 under autocast(float16): an overflowing scale skips the step (parameters
    unchanged, the scale drops, the gradients carry inf / NaN), and a few steps at a moderate scale stay finite and
    train.  make() -> a fresh model in its train recipe; trained(name) -> whether the parameter trains.

    That unscaled gradients do not depend on the scale is checked on the DeepLab head above, not here: two identical
    fp16 steps of these small whole models are not bitwise repeatable (the outputs of two runs with a torch trunk were
    1.5e-3 of max apart, the native trunk's squeeze-excite sums use float atomics), and ReLU and BatchNorm over a
    handful of images turn such differences into gradient differences of 5-60 % of max, whatever the scale."""
    from tests.test_encoder_train_gpu import loss_of

    def step(model, scaler, opt):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(5)
        with torch.autocast("cuda", dtype=torch.float16):
            loss = loss_of(model(image, inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"]))
        assert loss.dtype == torch.float32
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        torch.cuda.synchronize()
        return loss

    model = make()
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    step(model, scaler, opt)
    assert scaler.get_scale() < 2.0 ** 40
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    assert all(trained(k) for k in grads) and len(grads) > 20
    assert any(not bool(torch.isfinite(g).all()) for g in grads.values())
    assert all(torch.equal(p, before[k]) for k, p in model.named_parameters())

    model = make()
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    losses = [float(step(model, scaler, opt)) for _ in range(4)]
    assert all(torch.isfinite(torch.tensor(losses)))
    assert scaler.get_scale() >= 2.0 ** 10                  # at most a skipped step or two
    assert all(bool(torch.isfinite(p).all()) for p in model.parameters())
    moved = [k for k, p in model.named_parameters() if not torch.equal(p, before[k])]
    assert moved and all(trained(k) for k in moved)


def test_injected_torch_trunk_model_trains_under_autocast_with_grad_scaler():
    """the reference's recipe: model.train() with a torch trunk, precision=16"""
    from tests.test_encoder_train_gpu import LCFG, ConvTrunk, small_stp3
    torch.manual_seed(0)
    base, inp = small_stp3(ConvTrunk())
    image = gauss((1, 3, 2, 3, *LCFG.final_dim), 3).to(DEV)

    def make():
        m = copy.deepcopy(base)
        m.train()
        return m
    _model_scaler_checks(make, image, inp, lambda k: True)


def test_native_trunk_train_heads_recipe_under_autocast_with_grad_scaler():
    """the frozen native trunk: model.eval(); encoder.train_heads(); temporal model and decoder train"""
    from oracle import efficientnet_oracle as EO
    from tests.test_encoder_train_gpu import LCFG, small_stp3
    base, inp = small_stp3("native")
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=5), 'b4').eval()
    base.encoder.backbone.load_state_dict(ora.state_dict(), strict=True)
    base = base.to(DEV)
    image = gauss((1, 3, 2, 3, *LCFG.final_dim), 3).to(DEV)

    def make():
        m = copy.deepcopy(base)
        m.eval()
        m.encoder.train_heads()
        m.temporal_model.train()
        m.decoder.train()
        return m
    _model_scaler_checks(make, image, inp, lambda k: not k.startswith("encoder.backbone."))
