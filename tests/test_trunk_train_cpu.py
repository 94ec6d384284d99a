"""CPU: the opt-in train mode of the native EfficientNet trunk -- host logic (trainable flag, refusal text, state dict,
drop-connect rates and skip set, tape size), the fp64 train-mode restatement (tests/trunk_train_reference.py) against
the oracle modules, and the argument checks of the train-mode trunk entry points (fake pointers: nothing is launched)."""
import ctypes
import os

import pytest
import torch

from oracle import efficientnet_oracle as EO
from stp3_b200 import _lib
from stp3_b200.models import efficientnet as EN
from tests import trunk_train_reference as TR

FAKE = 1 << 20


@pytest.mark.parametrize("version,n_blocks,n_skip", [("b4", 22, 17), ("b0", 11, 6)])
def test_drop_connect_rates_and_skip_blocks(version, n_blocks, n_skip):
    _, _, specs = EN.trunk_table(version)
    assert len(specs) == n_blocks
    assert sum(s.skip for s in specs) == n_skip
    rates = EN.drop_connect_rates(len(specs))
    assert rates == [0.2 * i / n_blocks for i in range(n_blocks)] == TR.drop_rates(n_blocks)
    assert rates[0] == 0.0 and not specs[0].skip          # block 0 never draws
    net = EO.truncate(EO.EfficientNetOracle(version), version)
    assert [TR.is_skip(b.r) for b in net._blocks] == [s.skip for s in specs]


def test_trainable_is_opt_in_and_the_refusal_is_unchanged():
    t = EN.EfficientNetTrunk('b0')
    assert t.trainable is False
    with pytest.raises(NotImplementedError, match="eval-mode forward only") as e:
        t.train()
    assert str(e.value).startswith("EfficientNetTrunk: the sm_90a trunk implements the eval-mode forward only "
                                   "(BatchNorm folded into the kernels); training the trunk is not supported")
    assert "trainable=True" in str(e.value)
    assert not t.training
    t = EN.EfficientNetTrunk('b0', trainable=True)
    t.train()
    assert t.training and all(m.training for m in t.modules())
    t.eval()
    assert not any(m.training for m in t.modules())


@pytest.mark.parametrize("version", ["b4", "b0"])
def test_state_dict_is_the_same_with_and_without_trainable(version):
    a = EN.EfficientNetTrunk(version)
    b = EN.EfficientNetTrunk(version, trainable=True)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape and sa[k].dtype == sb[k].dtype for k in sa)
    b.load_state_dict(sa, strict=True)
    a.load_state_dict(sb, strict=True)
    ora = EO.truncate(EO.EfficientNetOracle(version), version)
    b.load_state_dict(ora.state_dict(), strict=True)


@pytest.mark.parametrize("version,H,W", [("b4", 224, 480), ("b0", 224, 480), ("b4", 64, 96), ("b0", 35, 51)])
def test_tape_size_formula(version, H, W):
    net = EO.truncate(EO.EfficientNetOracle(version), version)
    assert EN.trunk_tape_bytes(version, H, W) == 4 * TR.tape_elements(net, H, W)


def test_tape_size_of_the_nuscenes_batch():
    # b4 at 224 x 480: about 308 MB per image, 16.6 GB at M = 54 (3 samples x 3 frames x 6 cameras)
    per = EN.trunk_tape_bytes('b4', 224, 480)
    assert 3.0e8 < per < 3.2e8
    assert 1.6e10 < 54 * per < 1.7e10


def _oracle(version, seed=3):
    net = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=seed), version).double()
    return net


def test_restatement_matches_the_oracle_modules_without_drop_connect():
    net = _oracle('b0').train()
    x = torch.randn(3, 3, 40, 56, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    a = TR.trunk_forward(net, x)
    ref = EO.truncate(EO.init_random(EO.EfficientNetOracle('b0'), seed=3), 'b0').double().train()
    b = EO.endpoints(ref, x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_restatement_drop_connect_per_image():
    net = _oracle('b0').eval()
    blk_i = next(i for i, b in enumerate(net._blocks) if TR.is_skip(b.r) and i > 0)
    blk = net._blocks[blk_i]
    rate = TR.drop_rates(len(net._blocks))[blk_i]
    x = torch.randn(2, blk.r['cin'], 6, 7, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    full = TR.block_forward(blk, x, rate, None)
    got = TR.block_forward(blk, x, rate, torch.tensor([0.0, 1.0], dtype=torch.float64))
    assert torch.equal(got[0], x[0])                                  # dropped image: the skip alone
    torch.testing.assert_close(got[1] - x[1], (full[1] - x[1]) / (1 - rate), rtol=1e-12, atol=1e-12)


def test_masks_follow_torch_generator():
    net = _oracle('b4')
    torch.manual_seed(11)
    a = TR.draw_masks(net, 5, "cpu")
    torch.manual_seed(11)
    b = TR.draw_masks(net, 5, "cpu")
    assert list(a) == [i for i, blk in enumerate(net._blocks) if TR.is_skip(blk.r) and i > 0]
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert all(set(v.unique().tolist()) <= {0.0, 1.0} for v in a.values())


def test_images_that_require_grad_are_refused():
    t = EN.EfficientNetTrunk('b0', trainable=True).train()
    with pytest.raises(NotImplementedError, match="gradient with respect to the images is not computed"):
        t(torch.zeros(1, 3, 32, 32, requires_grad=True))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        t(torch.zeros(1, 3, 32, 32))


def test_train_mode_refuses_unsupported_batchnorm():
    for attr, val, msg in (("momentum", None, "momentum=None"), ("track_running_stats", False, "track_running_stats"),
                           ("affine", False, "affine=False")):
        t = EN.EfficientNetTrunk('b0', trainable=True).train()
        setattr(t._blocks[1]._bn1, attr, val)
        if attr == "track_running_stats":
            t._blocks[1]._bn1.running_mean = None
        with pytest.raises(NotImplementedError, match=msg):
            t.forward_train(_FakeCuda())


class _FakeCuda:
    """stands in for a CUDA image batch: forward_train checks BatchNorm modules before touching the data"""
    requires_grad = False
    is_cuda = True


def _lib_loaded():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


def _dw(**kw):
    d = dict(n_img=2, H=9, W=11, Ho=5, Wo=6, k=5, stride=2, pad_t=1, pad_l=1, C=24, in_cstride=24, out_cstride=24)
    d.update(kw)
    return ctypes.byref(_lib.DwDesc(**d))


def test_new_entry_points_refuse_bad_arguments():
    L = _lib_loaded()
    big = 1 << 40

    def refused(code, text):
        assert code == -1, code
        assert text.encode() in L.stp3_last_error(), L.stp3_last_error()

    refused(L.stp3_effnet_stem_raw(None, 1, 8, 8, 4, 4, 0, 0, FAKE, 32, FAKE, None), "null pointer")
    refused(L.stp3_effnet_stem_raw(FAKE, 1, 8, 8, 4, 4, 0, 0, FAKE, 65, FAKE, None), "cout must be in [1, 64]")
    refused(L.stp3_effnet_stem_raw(FAKE, 1, 8, 8, 4, 4, 3, 0, FAKE, 32, FAKE, None), "pad out of range")
    refused(L.stp3_effnet_stem_raw(FAKE, 0, 8, 8, 4, 4, 0, 0, FAKE, 32, FAKE, None), "non-positive dimension")
    refused(L.stp3_effnet_stem_wgrad(FAKE, 1, 8, 8, 4, 4, 0, 0, FAKE, 32, FAKE, FAKE, 8, None), "scratch smaller")
    refused(L.stp3_effnet_stem_wgrad(FAKE, 1, 8, 8, 4, 4, 0, 0, FAKE, 32, None, FAKE, big, None), "null pointer")
    assert L.stp3_effnet_stem_wgrad_scratch_bytes(1, 4, 4, 32) == 32 * 27 * 8
    for fn in (L.stp3_dw_fwd_raw, L.stp3_dw_dgrad):
        refused(fn(_dw(k=4), FAKE, FAKE, FAKE, None), "k must be 3 or 5")
        refused(fn(_dw(stride=3), FAKE, FAKE, FAKE, None), "stride must be 1 or 2")
        refused(fn(_dw(pad_t=5), FAKE, FAKE, FAKE, None), "pad out of range")
        refused(fn(_dw(in_cstride=16), FAKE, FAKE, FAKE, None), "row stride is smaller than C")
        refused(fn(_dw(Ho=0), FAKE, FAKE, FAKE, None), "non-positive dimension")
        refused(fn(_dw(), None, FAKE, FAKE, None), "null pointer")
        refused(fn(None, FAKE, FAKE, FAKE, None), "null descriptor")
    refused(L.stp3_dw_wgrad(_dw(), FAKE, FAKE, FAKE, FAKE, 8, None), "scratch smaller")
    refused(L.stp3_dw_wgrad(_dw(k=7), FAKE, FAKE, FAKE, FAKE, big, None), "k must be 3 or 5")
    assert L.stp3_dw_wgrad_scratch_bytes(_dw()) == 1 * 25 * 24 * 8
    refused(L.stp3_trunk_bn_act(FAKE, 10, 8, 3, None, None, None, None, 1, None, None, None, FAKE, None, None, 0, None),
            "bad argument")                                          # 10 pixels are not whole images of 3
    refused(L.stp3_trunk_bn_act(FAKE, 12, 8, 3, FAKE, None, FAKE, FAKE, 1, None, None, None, FAKE, None, None, 0, None),
            "mean needs invstd")
    refused(L.stp3_trunk_bn_act(FAKE, 12, 8, 3, None, None, None, None, 0, FAKE, None, None, None, FAKE, None, 64, None),
            "both bf16 planes")
    refused(L.stp3_trunk_bn_act(FAKE, 12, 80, 3, None, None, None, None, 0, FAKE, None, None, None, FAKE, FAKE, 64, None),
            "plane row stride smaller than C")
    refused(L.stp3_trunk_bn_act_bwd(FAKE, None, 12, 8, 3, None, None, None, None, 1, None, None, None, FAKE, None),
            "swish needs x")
    refused(L.stp3_trunk_bn_act_bwd(None, None, 12, 8, 3, None, None, None, None, 0, None, None, None, FAKE, None),
            "bad argument")
    refused(L.stp3_image_channel_dot(FAKE, FAKE, 2, 16, 8, FAKE, FAKE, 8, None), "scratch smaller")
    refused(L.stp3_image_channel_dot(FAKE, FAKE, 70000, 16, 8, FAKE, FAKE, big, None), "more than 65535 images")
    refused(L.stp3_image_channel_dot(FAKE, None, 2, 16, 8, FAKE, FAKE, big, None), "bad argument")
    assert L.stp3_image_channel_dot_scratch_bytes(2, 16, 8) == 2 * 8 * 8
    refused(L.stp3_se_bwd(FAKE, FAKE, FAKE, 2, 8, 0.5, FAKE, FAKE, 2, FAKE, FAKE, FAKE, None, FAKE, None), "null pointer")
    refused(L.stp3_se_bwd(FAKE, FAKE, FAKE, 2, 5000, 0.5, FAKE, FAKE, 2, FAKE, FAKE, FAKE, FAKE, FAKE, None),
            "bad dimensions")


# rows of the three partitioned reductions around every boundary of tests/trunk_train_reference.py's partition: one
# part, exact multiples of rows_per_part and one past them, the part cap and one past it, and the trunk's own sizes
_ROWS = sorted({1, 2, 255, 256, 257, 425, 511, 512, 513, 1023, 1024, 1025, 1275, 40320, 65535, 65536, 65537, 131071,
                131072, 131073, 161280, 262143, 262144, 262145, 282204, 10 ** 6})


def test_partition_mirror_matches_the_library_scratch_queries():
    """the scratch queries are host-only and size one fp64 partial per part, so they give the library's part counts"""
    L = _lib_loaded()
    for rows in _ROWS:
        for n_img, Ho, Wo in ((1, 1, rows), (1, rows, 1)) + (((rows // 6 // 7, 7, 1), (6, rows // 6, 1))
                                                             if rows % 42 == 0 else ()):
            for cout in (1, 48, 64):
                assert L.stp3_effnet_stem_wgrad_scratch_bytes(n_img, Ho, Wo, cout) == \
                    TR.stem_wgrad_parts(n_img, Ho, Wo) * cout * 27 * 8, (rows, cout)
            for k, C in ((3, 40), (5, 24)):
                d = _dw(n_img=n_img, H=Ho, W=Wo, Ho=Ho, Wo=Wo, k=k, stride=1, C=C, in_cstride=C + 8, out_cstride=C)
                assert L.stp3_dw_wgrad_scratch_bytes(d) == TR.dw_wgrad_parts(n_img, Ho, Wo) * k * k * C * 8, (rows, k)
        for n_img, C in ((1, 8), (7, 40)):
            assert L.stp3_image_channel_dot_scratch_bytes(n_img, rows, C) == n_img * TR.dot_parts(rows) * C * 8, rows


def test_partitions_of_the_trunk_steps():
    """the part counts the trunk-train contract's sources reach (stem output 17 x 25 at 35 x 51, 112 x 240 at 224 x 480)"""
    assert TR.stem_wgrad_parts(3, 17, 25) == 2 and TR.dot_parts(17 * 25) == 2 and TR.dw_wgrad_parts(3, 17, 25) == 3
    assert TR.part_features("dw", 3 * 17 * 25, 3, 512) == {"dw several parts"}
    assert TR.stem_wgrad_parts(6, 112, 240) == 158
    assert TR.part_features("stem", 6 * 112 * 240, 158, 1024) == {"stem several parts", "stem ragged last part"}
    assert TR.dw_wgrad_parts(6, 112, 240) == 256
    assert TR.part_features("dw", 6 * 112 * 240, 256, 512) == {"dw several parts", "dw part cap"}
    assert TR.dw_wgrad_parts(6, 56, 120) == 79
    assert TR.part_features("dw", 6 * 56 * 120, 79, 512) == {"dw several parts", "dw ragged last part"}
    assert TR.part_features("dot", 282204, 256, 256) == {"dot several parts", "dot ragged last part", "dot part cap"}
