"""GPU: the native EfficientNet trunk (stem, depthwise + squeeze-excite sums, gate folded into per-image projection
weights, swish / per-image-weight convolutions) against fp64, then the trunk, the encoder and STP3 from images."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet_oracle as EO
from oracle import torch_dense as TD
from stp3_b200 import dense
from stp3_b200.models import efficientnet as EN

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPLIT = 2.0 ** -17


def _hl(x64, cp):
    """(M, C, H, W) fp64 -> HL (M, 1, H, W, cp) and the exact fp64 value of the stored planes."""
    M, C, H, W = x64.shape
    hl = dense.from_f32(x64.float().to(DEV).unsqueeze(1), cp=cp)
    back = (hl.hi.double() + hl.lo.double())[:, 0, :, :, :C].permute(0, 3, 1, 2).cpu()
    return hl, back


def _val(hl, c, c_off=0):
    return (hl.hi.double() + hl.lo.double())[:, 0, :, :, c_off:c_off + c].permute(0, 3, 1, 2).cpu()


# (k, stride, (pad_t, pad_l), C, H, W).  The model passes the top / left pad of each static (before, after) pad pair:
# every depthwise launch of b4 and b0 at 224x480 (small batch) -- b4 k3 s2 (0, 0), k5 s2 (2, 2), b0 k5 s2 (1, 1), the
# stride-1 (k//2, k//2) -- then asymmetric pads, one-tile, odd and ragged sizes and 2-way to 15-way channel splits
DW_CASES = [(3, 1, (1, 1), 48, 112, 240), (3, 2, (0, 0), 144, 112, 240), (3, 1, (1, 1), 192, 56, 120),
            (5, 2, (2, 2), 192, 56, 120), (5, 1, (2, 2), 336, 28, 60), (3, 2, (0, 0), 336, 28, 60),
            (3, 1, (1, 1), 672, 14, 30), (5, 1, (2, 2), 672, 14, 30), (5, 1, (2, 2), 960, 14, 30),
            (3, 1, (1, 1), 32, 112, 240), (3, 2, (0, 0), 96, 112, 240), (5, 2, (1, 1), 144, 56, 120),
            (5, 1, (2, 2), 240, 28, 60), (3, 2, (0, 0), 240, 28, 60), (3, 1, (1, 1), 480, 14, 30),
            (5, 1, (2, 2), 480, 14, 30), (3, 1, (1, 1), 24, 112, 240), (3, 1, (1, 1), 144, 56, 120),
            (3, 2, (0, 1), 144, 112, 240), (5, 2, (1, 2), 144, 56, 120), (5, 1, (2, 2), 64, 8, 16),
            (3, 2, (0, 1), 40, 9, 17), (5, 2, (2, 2), 72, 23, 37)]


@pytest.mark.parametrize("k,s,pad,C,H,W", DW_CASES)
def test_depthwise_vs_fp64(k, s, pad, C, H, W):
    torch.manual_seed(k * 1000 + C + H)
    M = 3
    cp = dense.pad_to(C)
    x, x64 = _hl(torch.randn(M, C, H, W, dtype=torch.float64), cp)
    w = torch.randn(C, k * k, dtype=torch.float64) / k
    b = torch.randn(C, dtype=torch.float64) * 0.1
    wk = torch.zeros(k * k, cp, dtype=torch.float32)
    wk[:, :C] = w.t().float()
    bk = torch.zeros(cp, dtype=torch.float32)
    bk[:C] = b.float()
    Ho, Wo = EN.out_size(H, k, s, pad), EN.out_size(W, k, s, pad)
    # a wider output tensor filled with a sentinel: channels [cp, cp + 64) must stay untouched
    out = dense.HL(torch.full((M, 1, Ho, Wo, cp + 64), 3.0, dtype=torch.bfloat16, device=DEV),
                   torch.full((M, 1, Ho, Wo, cp + 64), 3.0, dtype=torch.bfloat16, device=DEV), C)
    sums = torch.empty((M, cp), dtype=torch.float32, device=DEV)
    dense.dw_conv(x, wk.to(DEV), bk.to(DEV), k, s, pad, (Ho, Wo), out=out, sums=sums)
    sums2 = torch.empty_like(sums)
    dense.dw_conv(x, wk.to(DEV), bk.to(DEV), k, s, pad, (Ho, Wo), out=out, sums=sums2)
    torch.cuda.synchronize()
    wq = wk[:, :C].double().t().reshape(C, 1, k, k)
    ref = F.silu(F.conv2d(F.pad(x64, (pad[1], pad[1] + 8, pad[0], pad[0] + 8)), wq, stride=s, groups=C)[:, :, :Ho, :Wo]
                 + bk[:C].double().view(1, C, 1, 1))
    got = _val(out, C)
    err = (got - ref).abs()
    assert (err <= SPLIT * ref.abs() + 1e-6 * ref.abs().max()).all(), err.max().item()
    assert torch.equal(sums, sums2), "squeeze-excite sums are not bitwise repeatable"
    s_ref = ref.sum((2, 3))
    assert ((sums[:, :C].double().cpu() - s_ref).abs() <= 1e-5 * s_ref.abs().max()).all()
    assert (sums[:, C:] == 0).all() and (_val(out, cp - C, C) == 0).all(), "padding channels are not zero"
    assert (out.hi[..., cp:] == 3.0).all() and (out.lo[..., cp:] == 3.0).all(), "bytes outside the window were written"


def _stem_ref(x64, w, b, pad):
    return F.silu(F.conv2d(F.pad(x64, (pad[1], pad[1] + 2, pad[0], pad[0] + 2)), w, stride=2) + b.view(1, -1, 1, 1))


def test_stem_vs_fp64():
    torch.manual_seed(3)
    M, H, W = 2, 224, 480
    x = torch.randn(M, 3, H, W, dtype=torch.float64)
    w = torch.randn(48, 3, 3, 3, dtype=torch.float64) * 0.3
    b = torch.randn(48, dtype=torch.float64) * 0.1
    pad = (0, 1)
    Ho, Wo = EN.out_size(H, 3, 2, pad), EN.out_size(W, 3, 2, pad)
    y = dense.effnet_stem(x.float().to(DEV), w.float().to(DEV).contiguous(), b.float().to(DEV), (Ho, Wo), pad)
    torch.cuda.synchronize()
    ref = _stem_ref(x.float().double(), w.float().double(), b.float().double(), pad)[:, :, :Ho, :Wo]
    err = (_val(y, 48) - ref).abs()
    assert (err <= SPLIT * ref.abs() + 1e-6 * ref.abs().max()).all(), err.max().item()
    assert (y.hi[..., 48:] == 0).all() and (y.lo[..., 48:] == 0).all()


@pytest.mark.parametrize("C,R,cout", [(960, 40, 160), (144, 6, 32), (336, 14, 112), (48, 12, 24)])
def test_gate_and_per_image_weights_vs_fp64(C, R, cout):
    torch.manual_seed(C + cout)
    n_img, hw = 5, 420
    cp = dense.pad_to(C)
    sums = torch.randn(n_img, cp, dtype=torch.float32) * hw * 0.3
    sums[:, C:] = 0
    w_r, b_r = torch.randn(R, C) / C ** 0.5, torch.randn(R) * 0.1
    w_e, b_e = torch.randn(C, R) / R ** 0.5, torch.randn(C) * 0.1
    w_p = torch.randn(cout, C) / C ** 0.5
    d = lambda t: t.float().contiguous().to(DEV)
    gate = torch.empty((n_img, C), dtype=torch.float32, device=DEV)
    w_img = dense.se_gate(d(sums), hw, C, d(w_r), d(b_r), d(w_e), d(b_e), d(w_p), gate=gate)
    torch.cuda.synchronize()
    m = sums[:, :C].double() / hw
    g_ref = torch.sigmoid(F.silu(m @ w_r.double().t() + b_r.double()) @ w_e.double().t() + b_e.double())
    assert (gate.double().cpu() - g_ref).abs().max() <= 1e-6
    assert w_img.shape == (n_img, dense.se_proj_weight_elems(C, cout))
    wi = w_img.cpu().double()
    off = 0
    for n0, n, bn in dense.se_chunks(cout):
        blk = wi[:, off:off + (cp // 64) * 2 * bn * 64].view(n_img, cp // 64, 2, bn, 64)
        val = (blk[:, :, 0] + blk[:, :, 1]).permute(0, 2, 1, 3).reshape(n_img, bn, cp)      # (img, row, k)
        ref = w_p[n0:n0 + n].double().unsqueeze(0) * g_ref.unsqueeze(1)
        assert ((val[:, :n, :C] - ref).abs() <= SPLIT * ref.abs() + 1e-6 * ref.abs().max()).all()
        assert (val[:, n:] == 0).all() and (val[:, :, C:] == 0).all()
        off += (cp // 64) * 2 * bn * 64


def _block_oracle(seed, r):
    blk = EO.MBConvBlock(r)
    net = torch.nn.Module()
    net.add_module("b", blk)
    EO.init_random(net, seed)
    return blk.eval()


@pytest.mark.parametrize("idx", [0, 2, 6, 9, 16, 21])
def test_block_expand_and_gated_projection_vs_fp64(idx):
    """One b4 block on the native path (swish expand convolutions, depthwise, gate, per-image projection with the skip
    as res_mode 1) against the fp64 restatement: the convolution contract's bar, <= 3e-5 of max."""
    _, _, rows = EO.block_table('b4')
    r = rows[idx]
    ora = _block_oracle(idx, r)
    nat = EN.EfficientNetTrunk('b4')
    nat._blocks[idx].load_state_dict(ora.state_dict(), strict=True)
    nat = nat.to(DEV)
    H, W = {0: (112, 240), 2: (112, 240), 6: (56, 120), 9: (28, 60), 16: (14, 30), 21: (14, 30)}[idx]
    torch.manual_seed(idx)
    x, x64 = _hl(torch.randn(4, r['cin'], H, W, dtype=torch.float64), dense.pad_to(r['cin']))
    gate = torch.empty((4, r['exp']), dtype=torch.float32, device=DEV)
    y = nat.forward_block(idx, x, gate=gate)
    y2 = nat.forward_block(idx, x)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = copy.deepcopy(ora).double()(x64)
    got = _val(y, r['cout'])
    e = (got - ref).abs().max().item() / ref.abs().max().item()
    print(f"block {idx}: {e:.2e} of max")
    assert e <= 3e-5, e
    assert torch.equal(y.hi, y2.hi) and torch.equal(y.lo, y2.lo), "the block is not bitwise repeatable"
    assert (y.hi[..., r['cout']:] == 0).all() and (y.lo[..., r['cout']:] == 0).all()


@pytest.fixture(scope="module")
def trunk_pair():
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle('b4'), seed=5), 'b4').eval()
    nat = EN.EfficientNetTrunk('b4')
    nat.load_state_dict(ora.state_dict(), strict=True)
    return ora, nat.to(DEV)


def test_trunk_endpoints_18_images_vs_fp64(trunk_pair):
    ora, nat = trunk_pair
    torch.manual_seed(0)
    x = torch.randn(18, 3, 224, 480)
    r3, r4 = nat(x.to(DEV))
    torch.cuda.synchronize()
    with torch.no_grad():
        o3, o4 = EO.endpoints(copy.deepcopy(ora).double().to(DEV), x.double().to(DEV))
    for name, got, ref in (("reduction_3", r3, o3), ("reduction_4", r4, o4)):
        e = (got.double() - ref).abs().max().item() / ref.abs().max().item()
        print(f"trunk {name}: {e:.2e} of max vs fp64")
        assert e <= 1e-3, (name, e)


def _stp3(backbone):
    from stp3_b200.config import get_cfg
    from stp3_b200.models.stp3 import STP3
    from stp3_b200.utils import synthetic as syn
    with torch.no_grad():
        model = STP3(get_cfg(), backbone=backbone)
        geo = {k: getattr(model, k).detach().clone() for k in ("frustum", "bev_resolution", "bev_start_position", "bev_dimension")}
        syn.init_exact(model, seed=0)
        for k, v in geo.items():
            getattr(model, k).copy_(v)
    return model.eval()


def test_encoder_and_stp3_from_images(trunk_pair):
    """Encoder(backbone="native") from images against the fp64 oracle trunk + fp64 heads; STP3.forward from images
    against the drop-in's forward_features fed with those fp64 encoder outputs (the lift / temporal / decoder path is
    pinned to fp64 elsewhere); the entry="images" graph replay at B = 4 reproduces eager
    and refuses a weight change after capture."""
    from stp3_b200.models.stp3 import GraphedPerception
    from stp3_b200.utils import synthetic as syn
    ora, _ = trunk_pair
    model = _stp3("native")
    assert model.encoder.native
    model.encoder.backbone.load_state_dict(ora.state_dict(), strict=True)
    model = model.to(DEV)
    inp = syn.lift_inputs(syn.CONFIGS["perceive"], 1, seed=3, random_pose=True)
    torch.manual_seed(1)
    image = torch.randn(1, 3, 6, 3, 224, 480)
    with torch.no_grad():
        enc64 = copy.deepcopy(model.encoder).cpu().double()
        o3, o4 = EO.endpoints(copy.deepcopy(ora).double().to(DEV), image.view(18, 3, 224, 480).double().to(DEV))
        f64, d64 = TD.encoder_heads(o3.cpu(), o4.cpu(), enc64)
        feat, depth = model.encoder(image.view(18, 3, 224, 480).to(DEV))
        torch.cuda.synchronize()
    for name, got, ref in (("features", feat, f64), ("depth", depth, d64)):
        e = (got.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
        print(f"encoder {name}: {e:.2e} of max vs fp64")
        assert e <= 1e-3, (name, e)
    with torch.no_grad():
        out = model(image.to(DEV), inp["intrinsics"], inp["extrinsics"], inp["future_egomotion"])
        ref = model.forward_features(f64.float().view(1, 3, 6, *f64.shape[1:]).to(DEV),
                                     d64.float().view(1, 3, 6, *d64.shape[1:]).to(DEV), inp["intrinsics"],
                                     inp["extrinsics"], inp["future_egomotion"])
        torch.cuda.synchronize()
    for k in ("segmentation", "pedestrian", "hdmap"):
        e = (out[k].double() - ref[k].double()).abs().max().item() / ref[k].abs().max().item()
        print(f"stp3 {k}: {e:.2e} of max")
        assert e <= 1e-3, (k, e)

    inp4 = syn.lift_inputs(syn.CONFIGS["perceive"], 4, seed=4, random_pose=True)
    image4 = torch.randn(4, 3, 6, 3, 224, 480)
    with torch.no_grad():
        eager = {k: v.clone() for k, v in model(image4.to(DEV), inp4["intrinsics"], inp4["extrinsics"],
                                                 inp4["future_egomotion"]).items() if torch.is_tensor(v)}
        g = GraphedPerception(model, 4, 6, entry="images")
        got = g(image4.to(DEV), None, inp4["intrinsics"], inp4["extrinsics"], inp4["future_egomotion"])
        torch.cuda.synchronize()
    # identical kernels and launch order; the trunk is deterministic, but the heads' pooling-branch spatial sums and
    # the lift-splat accumulate with float atomics, so only their summation order may differ (test_stp3_gpu's bar)
    d = (got["depth_prediction"] - eager["depth_prediction"]).abs().max() / eager["depth_prediction"].abs().max()
    assert d <= 1e-4, d.item()
    for k in ("segmentation", "pedestrian", "hdmap"):
        assert (got[k] - eager[k]).abs().max() <= 1e-4 * eager[k].abs().max(), k
    with torch.no_grad():
        model.encoder.backbone._blocks[3]._bn1.weight.mul_(1.5)
    with pytest.raises(RuntimeError, match="changed after the CUDA graph"):
        g(image4.to(DEV), None, inp4["intrinsics"], inp4["extrinsics"], inp4["future_egomotion"])


@pytest.mark.parametrize("name", ["trunk_b4_224x480", "trunk_b4_batch"])
def test_native_encoder_vs_reference_encoder_fixtures(name):
    """Encoder(backbone="native") against tests/golden/trunk_*.npz, made by the reference's own Encoder
    (delete_unused_layers, get_features_depth) around the fp32 restated trunk with the same seeded weights: both
    endpoints and both head outputs within 1e-3 of max."""
    import os
    import numpy as np
    from oracle import make_golden_trunk as MG
    from oracle.make_golden_dense import dense_input
    from stp3_b200.config import get_cfg
    from stp3_b200.models.encoder import Encoder
    g = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz")))
    img = dense_input(tuple(int(v) for v in g["shape"]), int(g["in_seed"]))
    with torch.no_grad():
        enc = MG.init_heads(Encoder(get_cfg().MODEL.ENCODER, D=48, backbone="native"))
        enc.backbone.load_state_dict(EO.truncate(MG.make_trunk(), 'b4').state_dict(), strict=True)
        enc = enc.eval().to(DEV)
        r3, r4 = enc.trunk(img.to(DEV))
        feat, depth = enc(img.to(DEV))
        torch.cuda.synchronize()
    for k, v in (("reduction_3", r3), ("reduction_4", r4), ("feature", feat), ("depth", depth)):
        ref = torch.from_numpy(g[k]).double()
        e = (v.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
        print(f"{name} {k}: {e:.2e} of max vs the reference Encoder")
        assert e <= 1e-3, (k, e)
