"""CPU: stp3_lift_splat_plan pins the kernel path of every lift-splat contract case (tests/lift_contract_cases.py), the
table reaches every path, and the backward refuses a tile it cannot hold before it launches anything.  Host only: fake,
never dereferenced device addresses."""
import os

import pytest

from stp3_b200 import _lib
from tests.lift_contract_cases import CASES, FAKE, PATHS, fake_desc, fake_plan, path_labels

NO_TMA = bool(int(os.environ.get("STP3_LIFT_NO_TMA", "0") or "0"))
skip_no_tma = pytest.mark.skipif(NO_TMA, reason="STP3_LIFT_NO_TMA turns the TMA scatter off (read once per process)")
DRIVER_FREE = ("tma_rules", "scatter_tw", "finalize", "finalize_vec", "finalize_smax", "finalize_lpp", "channel_groups")


@pytest.fixture(scope="module", autouse=True)
def library():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


@skip_no_tma
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_plan_pins_the_case_path(case):
    rc, plan = fake_plan(case)
    assert rc == 0, _lib.lib().stp3_last_error()
    assert {k: plan[k] for k in DRIVER_FREE} == case.plan


@skip_no_tma
def test_table_covers_every_path():
    reached = set()
    for case in CASES:
        reached |= path_labels(case, fake_plan(case)[1])
    assert PATHS <= reached, PATHS - reached
    # and the cases the GPU contract test needs for its pooling checks
    assert any(c.leftovers for c in CASES)
    tma = [c for c in CASES if c.plan["tma_rules"]]
    assert any(c.dims()["D"] % 16 for c in tma), "a TMA case with a partial last m-tile"
    assert any(c.dims()["Hf"] % 4 for c in tma), "a TMA case with padding rows"
    assert any(c.dims()["Hf"] == 32 for c in tma) and any(c.dims()["D"] == 256 for c in tma)
    assert any(not c.use_depth for c in tma)
    assert any(c.nhwc and c.C > 128 for c in tma) and any(not c.nhwc and c.C > 128 for c in tma)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_misaligned_feat_turns_only_the_tma_rule_off(case):
    rc, plan = fake_plan(case)
    rc4, plan4 = fake_plan(case, feat=FAKE + 4)
    assert rc == 0 and rc4 == 0
    assert plan4["tma_rules"] == 0 and plan4["scatter"] == 0
    assert {k: v for k, v in plan4.items() if k not in ("tma_rules", "scatter")} == \
           {k: v for k, v in plan.items() if k not in ("tma_rules", "scatter")}
    if case.use_depth:   # a misaligned depth map does the same
        assert fake_plan(case, depth=FAKE + 4)[1] == plan4


def test_plan_refuses_what_the_forward_refuses():
    L = _lib.lib()
    case = CASES[0]
    plan = _lib.LiftSplatPlan()
    cases = {
        "receptive field S=9": (fake_desc(case, S=9), 0, 0),
        "nz=2": (fake_desc(case, nz=2), 0, 0),
        "out_layout must be": (fake_desc(case), 3, 0),
        "frame mode writes fp32 channels-last": (fake_desc(case, f_begin=0, f_count=1), 0, 0),
        "peer outputs need frame mode": (fake_desc(case), 1, 1),
        "peer outputs need C in": (fake_desc(case, C=96, f_begin=0, f_count=1), 1, 1),
        "out_layout 2 needs C % 8 == 0": (fake_desc(case, C=33), 2, 0),
        "too large for one image column": (fake_desc(case, D=200, Hf=128), 0, 0),
    }
    for msg, (desc, layout, n_peers) in cases.items():
        assert L.stp3_lift_splat_plan(desc, FAKE, FAKE, layout, n_peers, plan) == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())
        assert L.stp3_lift_splat_fwd(desc, FAKE, FAKE, None, None, FAKE, 1 << 40, FAKE, layout, n_peers,
                                     None if not n_peers else (_lib.ctypes.c_void_p * 1)(FAKE), None) == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())
    assert L.stp3_lift_splat_plan(fake_desc(case, cam_M=None), FAKE, FAKE, 0, 0, plan) == -1
    assert b"stp3_lift_splat_plan: null pointer" in L.stp3_last_error()
    assert L.stp3_lift_splat_plan(fake_desc(case), FAKE, FAKE, 0, 0, None) == -1


def test_backward_refuses_an_oversized_tile_before_any_launch():
    """D = 96, Hf = 64: the forward takes it (one image column per CTA), the backward's tile does not fit in shared
    memory.  The refusal comes first: on a machine without a GPU any launch would fail with STP3_ECUDA (-3) instead."""
    L = _lib.lib()
    case = CASES[0]
    desc = fake_desc(case, D=96, Hf=64, Wf=6, C=64)
    plan = _lib.LiftSplatPlan()
    assert L.stp3_lift_splat_plan(desc, FAKE, FAKE, 0, 0, plan) == 0 and plan.scatter_tw == 1
    rc = L.stp3_lift_splat_bwd(desc, FAKE, FAKE, FAKE, FAKE, 1 << 40, FAKE, FAKE, None)
    assert rc == -1, (rc, L.stp3_last_error())
    assert b"too large for the backward tile" in L.stp3_last_error()
