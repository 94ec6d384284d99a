"""CPU: the EfficientNet trunk's block table, static pads, endpoints and state-dict surface (native module vs the torch
restatement in oracle/efficientnet_oracle.py, both against efficientnet-pytorch 0.7.0's published b4 table)."""
import pytest
import torch

from oracle import efficientnet_oracle as EO
from stp3_b200.models import efficientnet as EN

# (in, expanded, out, k, stride, SE width) of b4 blocks 0..21
B4 = ([(48, 48, 24, 3, 1, 12), (24, 24, 24, 3, 1, 6), (24, 144, 32, 3, 2, 6)] + [(32, 192, 32, 3, 1, 8)] * 3 +
      [(32, 192, 56, 5, 2, 8)] + [(56, 336, 56, 5, 1, 14)] * 3 + [(56, 336, 112, 3, 2, 14)] +
      [(112, 672, 112, 3, 1, 28)] * 5 + [(112, 672, 160, 5, 1, 28)] + [(160, 960, 160, 5, 1, 40)] * 5)
B4_STRIDE2_PADS = {2: (0, 1), 6: (2, 2), 10: (0, 1)}


def _native_rows(version):
    return [(s.cin, s.exp, s.cout, s.k, s.stride, s.se) for s in EN.trunk_table(version)[2]]


def test_b4_table_matches_the_published_block_table():
    stem, stem_pad, rows = EO.block_table('b4')
    assert stem == 48 and stem_pad == (0, 1)
    assert [(r['cin'], r['exp'], r['cout'], r['k'], r['s'], r['se']) for r in rows[:22]] == B4
    assert _native_rows('b4') == B4
    for i, r in enumerate(rows[:22]):
        want = B4_STRIDE2_PADS.get(i, (r['k'] // 2, r['k'] // 2))
        assert r['pad'] == want, (i, r['pad'], want)
        assert EN.trunk_table('b4')[2][i].pad == want
    assert EN.trunk_table('b4')[1] == (0, 1)


def test_b0_table_follows_the_same_rules():
    stem, stem_pad, rows = EO.block_table('b0')
    assert stem == 32 and stem_pad == (0, 1) and len(rows) == 16
    assert rows[3]['pad'] == (1, 2) and rows[3]['k'] == 5 and rows[3]['s'] == 2
    assert [(r['cin'], r['exp'], r['cout'], r['k'], r['s'], r['se']) for r in rows[:11]] == _native_rows('b0')
    assert [r['pad'] for r in rows[:11]] == [s.pad for s in EN.trunk_table('b0')[2]]


@pytest.mark.parametrize("version,hw,c3,c4", [('b4', (224, 480), 56, 160), ('b0', (224, 480), 40, 112)])
def test_endpoints_and_resolutions(version, hw, c3, c4):
    """reduction_3 / reduction_4 as the reference's get_features_depth picks them, at 1/8 and 1/16 of a 224x480 image;
    the native module's endpoint block and output sizes agree."""
    net = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=1), version).eval()
    with torch.no_grad():
        r3, r4 = EO.endpoints(net, torch.randn(1, 3, *hw))
    assert r3.shape == (1, c3, hw[0] // 8, hw[1] // 8) and r4.shape == (1, c4, hw[0] // 16, hw[1] // 16)
    nat = EN.EfficientNetTrunk(version)
    specs = EN.trunk_table(version)[2]
    assert specs[nat.endpoint].cout == c3 and specs[nat.endpoint + 1].stride == 2 and specs[-1].cout == c4
    h, w = (EN.out_size(n, 3, 2, nat.stem_pad) for n in hw)
    sizes = []
    for s in specs:
        h, w = EN.out_size(h, s.k, s.stride, s.pad), EN.out_size(w, s.k, s.stride, s.pad)
        sizes.append((h, w))
    assert sizes[nat.endpoint] == (hw[0] // 8, hw[1] // 8) and sizes[-1] == (hw[0] // 16, hw[1] // 16)


@pytest.mark.parametrize("version", ['b4', 'b0'])
def test_state_dict_keys_and_shapes_match_and_load_strict(version):
    ora = EO.truncate(EO.init_random(EO.EfficientNetOracle(version), seed=2), version)
    nat = EN.EfficientNetTrunk(version)
    a, b = ora.state_dict(), nat.state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape for k in a)
    assert not any(k.startswith(('_conv_head', '_bn1', '_fc')) for k in b)
    nat.load_state_dict(a, strict=True)
    ora.load_state_dict(nat.state_dict(), strict=True)
    assert all(torch.equal(a[k], nat.state_dict()[k]) for k in a)
    assert all(m.eps == 1e-3 for m in nat.modules() if isinstance(m, torch.nn.BatchNorm2d))


def test_native_trunk_refuses_train_mode():
    nat = EN.EfficientNetTrunk('b0')
    assert not nat.training
    with pytest.raises(NotImplementedError, match="eval-mode"):
        nat.train()
    nat.eval()


def test_launches_per_block():
    """Expand chunks of <= 128 columns, depthwise + its sum reduction, gate + weight scaling, projection chunks."""
    n = EN.EfficientNetTrunk('b4').launches_per_block()
    assert n[0] == 0 + 2 + 2 + 1 and n[2] == 2 + 2 + 2 + 1 and n[21] == 8 + 2 + 2 + 2
    assert sum(n) == 214


def _golden(name):
    import os
    import numpy as np
    return dict(np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz")))


@pytest.mark.parametrize("name", ["trunk_b4_224x480", "trunk_b4_batch"])
def test_restatement_reproduces_the_reference_encoder_fixtures(name):
    """tests/golden/trunk_*.npz come from the reference's own Encoder (delete_unused_layers, get_features_depth) around
    the fp32 restated trunk (oracle/make_golden_trunk.py).  The restatement's endpoints and the heads evaluated on them
    reproduce them."""
    from oracle import make_golden_trunk as MG
    from oracle import torch_dense as TD
    from oracle.make_golden_dense import dense_input
    from stp3_b200.config import get_cfg
    from stp3_b200.models.encoder import Encoder
    g = _golden(name)
    img = dense_input(tuple(int(v) for v in g["shape"]), int(g["in_seed"]))
    with torch.no_grad():
        trunk = EO.truncate(MG.make_trunk(), 'b4')
        r3, r4 = EO.endpoints(trunk, img)
        enc = MG.init_heads(Encoder(get_cfg().MODEL.ENCODER, D=48, backbone="native")).eval()
        feat, depth = TD.encoder_heads(r3, r4, enc)
    for k, v in (("reduction_3", r3), ("reduction_4", r4), ("feature", feat), ("depth", depth)):
        ref = torch.from_numpy(g[k])
        assert v.shape == ref.shape, k
        assert (v - ref).abs().max() <= 1e-5 * ref.abs().max(), k


@pytest.mark.parametrize("name", ["trunk_b4_224x480", "trunk_b4_batch"])
def test_reference_encoder_regenerates_the_fixtures(name):
    """The fixtures are what the unmodified reference Encoder computes today (needs the reference install)."""
    from oracle import make_golden_trunk as MG
    from oracle.make_golden_dense import dense_input
    from oracle.ref_loader import reference_available, load_reference
    if not reference_available():
        pytest.skip("the reference install (oracle/_ref or STP3_REFERENCE_ROOT) is not present")
    g = _golden(name)
    img = dense_input(tuple(int(v) for v in g["shape"]), int(g["in_seed"]))
    with torch.no_grad():
        out = MG.run(MG.reference_encoder(load_reference()), img)
    for k, v in zip(("reduction_3", "reduction_4", "feature", "depth"), out):
        assert torch.equal(v, torch.from_numpy(g[k])), k
