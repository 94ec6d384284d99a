"""The lift-splat contract cases (tests/test_lift_splat_plan_cpu.py, tests/test_lift_splat_contract_gpu.py): small,
non-square BEV grids whose pillar counts are not multiples of a finalize CTA's 32 / 128 / 64 / 32 pillars, each case
pinned to the kernel path stp3_lift_splat_plan chooses for it.  PATHS names every path the table must reach."""
import ctypes
from dataclasses import dataclass, field
from typing import Optional, Tuple

from stp3_b200 import _lib
from stp3_b200.utils import synthetic as syn

FAKE = 1 << 20        # a non-null, 256-byte aligned address: the plan query never dereferences it

XB, YB = (-11.25, 11.25, 0.5), (-9.5, 9.5, 0.5)          # 45 x 38 = 1710 pillars, power-of-two resolution
XB2, YB2 = (-6.1, 6.1, 0.2), (-4.5, 4.5, 0.2)            # 0.2 m (true division), non-square


@dataclass
class Case:
    name: str
    D_bound: Tuple[float, float, float]
    final_dim: Tuple[int, int]          # image size; the feature map is final_dim // 8
    C: int
    S: int
    N: int = 2
    B: int = 1
    xb: Tuple[float, float, float] = XB
    yb: Tuple[float, float, float] = YB
    seed: int = 0
    random_pose: bool = True
    nhwc: bool = False                  # channels-last features
    use_depth: bool = True
    out_layout: int = 0                 # 0 (B,S,C,X,Y) fp32, 1 (B,S,X,Y,C) fp32, 2 bf16 hi/lo planes
    pool_sum: bool = False
    frames: Optional[Tuple[int, int]] = None   # (f_begin, f_count): frame-sharded call, raw splats
    n_peers: int = 0                    # frame mode: number of gathered buffers the finalize stores into
    leftovers: bool = False             # the ranks must give (depth, column) pairs of 2-4 and of more than 4 pillars
    plan: dict = field(default_factory=dict)   # expected tma_rules, scatter_tw, finalize, finalize_vec / smax / lpp, channel_groups

    def config(self) -> syn.LiftSplatConfig:
        return syn.LiftSplatConfig(x_bound=self.xb, y_bound=self.yb, d_bound=self.D_bound, final_dim=self.final_dim,
                                   out_channels=self.C, n_cameras=self.N, receptive_field=self.S)

    def dims(self):
        cfg = self.config()
        Hf, Wf = cfg.feat_hw
        return dict(D=cfg.n_depth, Hf=Hf, Wf=Wf)


def P(tma, tw, fin, vec, smax, lpp, groups):
    return dict(tma_rules=tma, scatter_tw=tw, finalize=fin, finalize_vec=vec, finalize_smax=smax, finalize_lpp=lpp,
                channel_groups=groups)


LPP_FIN = 0   # finalize: lane-per-pillar kernel
CL_FIN = 1    # finalize: channels-last kernel

CASES = [
    # ---- TMA-staged scatter
    # D = 41: partial last m-tile (41 = 2 x 16 + 9, depths 2-10 m, all inside the grid); Hf = 7: padded rows of HP = 8
    # and an all-padding second k-step
    Case("tma_d41_hf7", (2.0, 10.2, 0.2), (56, 96), 64, 2, out_layout=0, pool_sum=True,
         plan=P(1, 4, LPP_FIN, 1, 4, 0, 1)),
    # D = 256 (the limit), 0.1 m depth steps, Hf = 4
    Case("tma_d256", (1.0, 26.6, 0.1), (32, 64), 64, 1, out_layout=1, pool_sum=True, plan=P(1, 4, CL_FIN, 0, 4, 4, 1)),
    # Hf = 32 (the limit, both k-steps full), two channel chunks, NCHW and NHWC
    Case("tma_hf32_c128_nchw", (2.0, 50.0, 1.0), (256, 64), 128, 4, N=1, out_layout=2, pool_sum=True,
         plan=P(1, 4, CL_FIN, 0, 4, 8, 1)),
    Case("tma_hf32_c128_nhwc", (2.0, 50.0, 1.0), (256, 64), 128, 1, nhwc=True, out_layout=1, pool_sum=True,
         plan=P(1, 4, CL_FIN, 0, 4, 8, 1)),
    # three channel chunks: the feature barrier's phase bit wraps; D = 33 (a one-row last m-tile), Hf = 16; S = 5 on
    # the lane-per-pillar kernel
    Case("tma_c192_nhwc_s5", (2.0, 8.6, 0.2), (128, 64), 192, 5, N=1, nhwc=True, out_layout=1, pool_sum=True,
         plan=P(1, 4, LPP_FIN, 1, 8, 0, 3)),
    Case("tma_c192_nchw", (2.0, 8.6, 0.2), (128, 64), 192, 1, out_layout=0, plan=P(1, 4, LPP_FIN, 1, 4, 0, 3)),
    # no depth distribution: the depth map is never fetched; D = 24
    Case("tma_no_depth", (2.0, 6.8, 0.2), (64, 96), 64, 4, use_depth=False, out_layout=2, pool_sum=True,
         plan=P(1, 4, CL_FIN, 0, 4, 4, 1)),
    # S = 8 (7 chained poses: the shared-memory pose walk), hi/lo output on the lane-per-pillar kernel; D = 20
    Case("tma_s8", (2.0, 10.0, 0.4), (48, 64), 64, 8, out_layout=2, pool_sum=True, plan=P(1, 4, LPP_FIN, 1, 8, 0, 1)),
    # 0.2 m grid, tilted cameras: (depth, column) pairs over 2-4 pillars (tensor-core passes) and over more (scalar walk)
    Case("tma_leftovers", (2.0, 18.0, 1.0), (224, 64), 128, 2, N=3, xb=XB2, yb=YB2, seed=3, out_layout=0,
         pool_sum=True, leftovers=True, plan=P(1, 4, LPP_FIN, 1, 4, 0, 2)),
    # D = 1, Hf = 1
    Case("tma_d1_hf1", (2.0, 3.0, 1.0), (8, 64), 64, 2, out_layout=0, plan=P(1, 4, LPP_FIN, 1, 4, 0, 1)),
    # ---- generic scatter
    # Hf = 33: one past the TMA limit, two row chunks (the second holds one row)
    Case("gen_hf33", (2.0, 50.0, 1.0), (264, 64), 64, 1, N=1, out_layout=2, pool_sum=True,
         plan=P(0, 2, CL_FIN, 0, 4, 4, 1)),
    # Hf = 40: a partial second row chunk; C = 32 on the channels-last kernel (LPP 2)
    Case("gen_hf40_c32", (2.0, 50.0, 1.0), (320, 64), 32, 4, N=1, out_layout=1, pool_sum=True,
         plan=P(0, 2, CL_FIN, 0, 4, 2, 1)),
    # D = 96, Hf = 64: one image column per CTA
    Case("gen_tw1", (2.0, 98.0, 1.0), (512, 48), 64, 1, N=1, out_layout=0, pool_sum=True,
         plan=P(0, 1, LPP_FIN, 1, 4, 0, 1)),
    # C = 96: a partial second channel chunk in the scatter and in the finalize's channel groups; 0.2 m grid
    Case("gen_c96", (2.0, 26.0, 1.0), (64, 96), 96, 3, xb=XB2, yb=YB2, out_layout=0, pool_sum=True,
         plan=P(0, 4, LPP_FIN, 1, 4, 0, 2)),
    # C = 33 (odd: scalar atomics, scalar finalize), Wf = 10 (no TMA), NCHW and NHWC, S = 6
    Case("gen_c33_nchw", (2.0, 18.0, 1.0), (64, 80), 33, 2, out_layout=0, pool_sum=True,
         plan=P(0, 4, LPP_FIN, 0, 4, 0, 1)),
    Case("gen_c33_nhwc_s6", (2.0, 18.0, 1.0), (64, 80), 33, 6, nhwc=True, out_layout=1, pool_sum=True,
         plan=P(0, 4, LPP_FIN, 0, 8, 0, 1)),
    # D = 257: one past the TMA limit
    Case("gen_d257", (1.0, 26.7, 0.1), (32, 64), 32, 1, out_layout=2, pool_sum=True, plan=P(0, 4, CL_FIN, 0, 4, 2, 1)),
    # C = 8 with 8-channel vector loads and a single warp per CTA, S = 7
    Case("gen_c8_s7", (2.0, 18.0, 1.0), (48, 64), 8, 7, out_layout=1, pool_sum=True, plan=P(0, 4, LPP_FIN, 1, 8, 0, 1)),
    # ---- frame-sharded calls: raw splats of frames [f_begin, f_begin + f_count) of B * S
    Case("frames_c64", (2.0, 18.0, 1.0), (48, 64), 64, 3, B=2, frames=(1, 4), out_layout=1,
         plan=P(1, 4, CL_FIN, 0, 4, 4, 1)),
    Case("frames_peers_c32", (2.0, 18.0, 1.0), (48, 64), 32, 3, B=2, frames=(2, 3), n_peers=2, out_layout=1,
         plan=P(0, 4, CL_FIN, 0, 4, 2, 1)),
    Case("frames_peers_c128", (2.0, 18.0, 1.0), (48, 64), 128, 2, B=2, frames=(1, 2), n_peers=2, out_layout=1,
         plan=P(1, 4, CL_FIN, 0, 4, 8, 1)),
]
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def path_labels(case: Case, plan: dict):
    """The paths a case with this plan reaches: the scatter kernel and its layout, the finalize kernel and its
    variant, the output layout."""
    out = set()
    if plan["tma_rules"]:
        out.add("scatter TMA " + ("NHWC" if case.nhwc else "NCHW"))
    else:
        out.add(f"scatter generic TW{plan['scatter_tw']}")
    if plan["finalize"] == CL_FIN:
        out.add(f"finalize channels-last LPP{plan['finalize_lpp']}" + (" peers" if case.n_peers else ""))
    else:
        out.add(f"finalize lane-per-pillar {'VEC' if plan['finalize_vec'] else 'scalar'} SMAX{plan['finalize_smax']}")
    out.add(f"out_layout {case.out_layout}")
    return out


PATHS = {"scatter TMA NCHW", "scatter TMA NHWC", "scatter generic TW4", "scatter generic TW2", "scatter generic TW1",
         "finalize lane-per-pillar VEC SMAX4", "finalize lane-per-pillar VEC SMAX8",
         "finalize lane-per-pillar scalar SMAX4", "finalize lane-per-pillar scalar SMAX8",
         "finalize channels-last LPP2", "finalize channels-last LPP4", "finalize channels-last LPP8",
         "finalize channels-last LPP2 peers", "finalize channels-last LPP8 peers",
         "out_layout 0", "out_layout 1", "out_layout 2"}


def fake_desc(case: Case, **kw):
    """stp3_lift_splat_desc of the case with fake geometry pointers (for the host-only plan query)."""
    d = case.dims()
    cfg = case.config()
    nx, ny = cfg.bev_xy
    f0, fc = case.frames or (0, 0)
    f = dict(cam_M=FAKE, cam_t=FAKE, ego_R=FAKE, ego_t=FAKE, xs=FAKE, ys=FAKE, ds=FAKE,
             bev_off=(ctypes.c_float * 3)(cfg.x_bound[0], cfg.y_bound[0], -10.0),
             bev_res=(ctypes.c_float * 3)(cfg.x_bound[2], cfg.y_bound[2], 20.0), nx=nx, ny=ny, nz=1,
             discount=cfg.discount, B=case.B, S=case.S, N=case.N, D=d["D"], Hf=d["Hf"], Wf=d["Wf"], C=case.C,
             feat_layout=int(case.nhwc), use_depth_distribution=int(case.use_depth), f_begin=f0, f_count=fc)
    f.update(kw)
    return _lib.LiftSplatDesc(**f)


def fake_plan(case: Case, feat=FAKE, depth=FAKE):
    """(return code, plan dict) of stp3_lift_splat_plan for the case at the given feat / depth_logits addresses."""
    plan = _lib.LiftSplatPlan()
    rc = _lib.lib().stp3_lift_splat_plan(fake_desc(case), feat, depth, case.out_layout, case.n_peers, ctypes.byref(plan))
    return rc, {name: getattr(plan, name) for name, _ in _lib.LiftSplatPlan._fields_}
