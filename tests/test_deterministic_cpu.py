"""CPU: a numpy model of the lift-splat's deterministic mode (64-bit fixed point, DESIGN.md §3.14) -- the per-frame
scale rule, rounding to the grid, the int64 sum, the conversion back to fp32 and the fp32 discount recurrence -- the
overflow bound, and the refusals and workspace formula of the new C entry points.  tests/test_deterministic_gpu.py
checks the kernels against fixed_point_bev bit for bit."""
import ctypes
import math
from fractions import Fraction

import numpy as np

from stp3_b200 import _lib
from tests.test_abi import FAKE, lift_desc

F32_MAX = float(np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------------ the model
def f32_bits(x) -> int:
    return int(np.float32(x).view(np.uint32))


def ceil_log2(x: float) -> int:
    """ceil(log2 x) for a finite float x > 0, exactly"""
    f, e = math.frexp(x)            # x = f * 2^e, 0.5 <= f < 1
    return e - 1 if f == 0.5 else e


def frame_max(feat_frame: np.ndarray) -> np.float32:
    """m_f: the largest finite |feature| of a frame (0 when there is none)"""
    a = np.abs(np.asarray(feat_frame, np.float32).reshape(-1))
    a = a[np.isfinite(a)]
    return np.float32(a.max()) if a.size else np.float32(0)


def ceil_log2_points(points: int) -> int:
    return (points - 1).bit_length()


def frame_exponent(m: np.float32, points: int) -> int:
    """k_f = 62 - (ceil(log2 m_f) + ceil(log2 points)); 0 for an all-zero frame"""
    return 0 if m == 0 else 62 - (ceil_log2(float(m)) + ceil_log2_points(points))


def quantize(partial: np.ndarray, k: int) -> np.ndarray:
    """fp32 partials -> int64 multiples of 2^-k, rounded to nearest even (__double2ll_rn)"""
    return np.rint(np.asarray(partial, np.float32).astype(np.float64) * 2.0 ** k).astype(np.int64)


def to_f32(q: np.ndarray, k: int) -> np.ndarray:
    """__double2float_rn((double)q * 2^-k)"""
    return (np.asarray(q, np.int64).astype(np.float64) * 2.0 ** -k).astype(np.float32)


def recurrence(frames: np.ndarray, discount: np.float32) -> np.ndarray:
    """out[t] = fp32(fp32(out[t-1] * discount) + v[t]) over axis 0"""
    out = np.empty_like(frames, dtype=np.float32)
    acc = np.zeros(frames.shape[1:], np.float32)
    for t in range(frames.shape[0]):
        acc = (acc * discount).astype(np.float32) + frames[t]
        out[t] = acc
    return out


def column_partials(rows: np.ndarray, r: np.ndarray):
    """(pillar, fp32 partial over C) flushes of one image column with probability 1: one add chain over the valid rows
    when they all share a pillar, else one chain per run of equal ranks (lift_splat_scatter_kernel's two paths)"""
    valid = r >= 0
    if not valid.any():
        return []
    if len(set(r[valid].tolist())) == 1:
        a = np.zeros(rows.shape[1], np.float32)
        for h in np.flatnonzero(valid):
            a = a + rows[h]
        return [(int(r[valid][0]), a)]
    out, cur, a = [], -1, np.zeros(rows.shape[1], np.float32)
    for h in range(len(r)):
        if r[h] != cur:
            if cur >= 0:
                out.append((cur, a))
            cur, a = int(r[h]), np.zeros(rows.shape[1], np.float32)
        a = a + rows[h]
    if cur >= 0:
        out.append((cur, a))
    return out


def fixed_point_bev(feat: np.ndarray, ranks: np.ndarray, nvox: int, discount: np.float32) -> np.ndarray:
    """(B,S,nvox,C) output of the deterministic lift-splat with use_depth_distribution = 0 for feat (B,S,N,C,Hf,Wf)
    and the kernel's ranks (B,S,N,D,Hf,Wf), image rows in one chunk (Hf <= 32)"""
    B, S, N, C, Hf, Wf = feat.shape
    D = ranks.shape[3]
    assert Hf <= 32
    raw = np.zeros((B, S, nvox, C), np.float32)
    for b in range(B):
        for t in range(S):
            k = frame_exponent(frame_max(feat[b, t]), N * D * Hf * Wf)
            grid = np.zeros((nvox, C), np.int64)
            for n in range(N):
                img = feat[b, t, n].transpose(1, 2, 0)          # (Hf, Wf, C)
                for d in range(D):
                    for w in range(Wf):
                        for rank, a in column_partials(img[:, w], ranks[b, t, n, d, :, w]):
                            grid[rank] += quantize(a, k)
            raw[b, t] = to_f32(grid, k)
    return np.stack([recurrence(raw[b], discount) for b in range(B)])


# ------------------------------------------------------------------------------------------------ scale rule
def test_ceil_log2_matches_exact_arithmetic():
    rng = np.random.default_rng(0)
    xs = [np.float32(2.0 ** e) for e in range(-149, 128)] + list(rng.random(200, np.float32) * 1e6) + \
         [np.float32(v) for v in (1.5, 3.0, 0.75, F32_MAX, np.finfo(np.float32).tiny, 1e-45, 3e-45)]
    for x in xs:
        x = float(x)
        k = ceil_log2(x)
        assert Fraction(2) ** (k - 1) < Fraction(x) <= Fraction(2) ** k, x


def test_scale_rule_edge_cases():
    points = 6 * 48 * 28 * 60
    lp = ceil_log2_points(points)
    assert lp == 19
    assert frame_exponent(np.float32(0), points) == 0                               # all-zero frame
    assert frame_exponent(np.float32(1.0), points) == 62 - 19
    assert frame_exponent(np.float32(1.5), points) == 62 - 1 - 19
    sub = np.uint32(1).view(np.float32)                                             # 2^-149
    assert frame_exponent(sub, points) == 62 + 149 - 19
    assert frame_exponent(np.uint32(3).view(np.float32), points) == 62 + 147 - 19   # 3 * 2^-149
    assert frame_exponent(np.float32(F32_MAX), points) == 62 - 128 - 19             # negative: coarser than 1
    # non-finite values are left out of m_f
    f = np.array([1.0, -7.5, np.nan, np.inf, -np.inf, 2.0], np.float32)
    assert frame_max(f) == np.float32(7.5)
    assert frame_max(np.array([np.nan, np.inf], np.float32)) == 0
    # every exponent the rule gives keeps the scale 2^k a normal double and 2^-k representable for the conversion
    for m in (sub, np.float32(F32_MAX)):
        for pts in (1, points, 2 ** 40):
            k = frame_exponent(m, pts)
            assert -1022 <= k <= 1023 and -1022 <= -k <= 1023


def test_overflow_bound_worst_case():
    """Every point of the largest admissible frame adds m_f (times a probability that rounding may lift to 1 + 2^-23)
    into ONE pillar: the int64 sum stays below 2^63.  The frame is bounded far beyond what the kernels admit (D <= 256
    on the TMA path, a CTA grid below 2^31): 2^40 points."""
    for m in (np.uint32(1).view(np.float32), np.float32(1.0), np.float32(1.0 + 2 ** -23), np.float32(3.0),
              np.float32(F32_MAX)):
        for points in (1, 2, 3, 1000, 6 * 48 * 28 * 60, 2 ** 40 - 1, 2 ** 40):
            k = frame_exponent(m, points)
            worst = float(np.float32(m)) * (1 + 2.0 ** -23)          # one point's largest partial
            q = round(Fraction(worst) * Fraction(2) ** k)            # its grid value (an upper bound of the rounding)
            assert points * q < 2 ** 63, (m, points, k)
            assert points * q <= 2 ** 62 * (1 + 2 ** -22), (m, points, k)


# ------------------------------------------------------------------------------------------------ rounding and sums
def test_rounding_to_the_grid_is_nearest():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(10000) * 10).astype(np.float32)
    for k in (-3, 0, 7, 20, 43):
        q = quantize(x, k)
        err = np.abs(q.astype(np.float64) * 2.0 ** -k - x.astype(np.float64))
        assert err.max() <= 2.0 ** (-k - 1)
    # ties go to even, like __double2ll_rn
    assert quantize(np.array([0.5, 1.5, 2.5, -0.5, -1.5], np.float32), 0).tolist() == [0, 2, 2, 0, -2]
    # truncation would lose up to a full step: 0.75 -> 0, not 1
    assert quantize(np.array([0.75, -0.75], np.float32), 0).tolist() == [1, -1]


def test_int64_sum_is_order_independent_and_within_one_ulp():
    rng = np.random.default_rng(2)
    for trial in range(20):
        n = int(rng.integers(1, 4000))
        parts = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4)).astype(np.float32)
        m = np.float32(np.abs(parts).max())
        k = frame_exponent(m, n)
        q = quantize(parts, k)
        total = int(q.sum())
        assert total == int(q[rng.permutation(n)].sum())            # any arrival order
        assert abs(total) < 2 ** 62
        got = to_f32(np.array([total]), k)[0]
        exact_grid = Fraction(total) * Fraction(2) ** -k            # the exact sum of the grid-rounded partials
        ulp = Fraction(float(np.spacing(np.abs(got)))) if got != 0 else Fraction(2) ** -149
        assert abs(Fraction(float(got)) - exact_grid) <= ulp
        exact = sum(Fraction(float(p)) for p in parts)               # rounding to the grid adds <= 2^-(k+1) per part
        assert abs(exact_grid - exact) <= n * Fraction(2) ** (-k - 1)


def test_recurrence_is_the_fp32_chain():
    v = np.array([[1.0], [2.0 ** -30], [3.0]], np.float32)
    out = recurrence(v, np.float32(0.5))
    assert out[:, 0].tolist() == [1.0, np.float32(np.float32(0.5) + np.float32(2.0 ** -30)), np.float32(3.25)]
    nan = recurrence(np.array([[0.0], [np.nan], [1.0]], np.float32), np.float32(0.5))
    assert nan[0, 0] == 0 and np.isnan(nan[1:, 0]).all()             # a poisoned pillar stays NaN in later frames


def test_host_model_on_a_tiny_frame():
    """Two cameras, two depth bins, three rows, one column: a shared-pillar column (one chain, masked rows skipped) and
    a split column (one chain per run)."""
    feat = np.zeros((1, 1, 2, 2, 3, 1), np.float32)
    feat[0, 0, 0, :, :, 0] = [[1.0, 2.0, 4.0], [0.5, 0.25, 0.125]]
    feat[0, 0, 1, :, :, 0] = [[-1.0, 3.0, 1.0], [1.0, 1.0, 1.0]]
    ranks = np.full((1, 1, 2, 2, 3, 1), -1, np.int32)
    ranks[0, 0, 0, 0, :, 0] = [5, -1, 5]            # rows 0 and 2 into pillar 5
    ranks[0, 0, 1, 1, :, 0] = [2, 3, 2]             # runs: 2, 3, 2
    out = fixed_point_bev(feat, ranks, 8, np.float32(0.5))[0, 0]
    assert out[5].tolist() == [5.0, 0.625]
    assert out[2].tolist() == [0.0, 2.0] and out[3].tolist() == [3.0, 1.0]
    assert not out[[0, 1, 4, 6, 7]].any()


# ------------------------------------------------------------------------------------------------ C ABI
def _al(x):
    return (x + 255) // 256 * 256


def test_det_workspace_formula():
    L = _lib.lib()
    frames, nvox, C = 3, 200 * 200, 64
    want = (_al(frames * nvox * C * 8) + _al(frames * nvox) + _al(1250 * frames * C * 4) + _al(frames * 4)
            + _al(frames * ((nvox + 31) // 32) * 4) + _al(frames * 16 * C * 4))
    assert L.stp3_lift_splat_det_workspace_bytes(lift_desc()) == want
    for kw in ({}, dict(f_begin=1, f_count=2), dict(C=33, nx=45, ny=38), dict(B=4, S=3, C=64)):
        d = lift_desc(**kw)
        assert L.stp3_lift_splat_det_workspace_bytes(d) >= L.stp3_lift_splat_workspace_bytes(d)
    assert L.stp3_lift_splat_det_workspace_bytes(lift_desc(B=0)) == 0
    assert L.stp3_lift_splat_det_workspace_bytes(None) == 0
    # perceive (B = 4, S = 3, 200 x 200, C = 64): 246 MB of int64 grid; the stress shape per GPU: 6.6 GB
    assert 4 * 3 * nvox * 64 * 8 == 245_760_000
    assert 8 * 5 * 400 * 400 * 128 * 8 == 6_553_600_000


def test_det_entry_refusals():
    L = _lib.lib()

    def fwd(desc, ranks_out=None, out_layout=0, n_peers=0, ws_bytes=1 << 40):
        peers = (ctypes.c_void_p * 1)(FAKE) if n_peers else None
        return L.stp3_lift_splat_fwd_det(desc, FAKE, FAKE, ranks_out, None, FAKE, ws_bytes, FAKE, out_layout, n_peers,
                                         peers, None)

    cases = {
        "receptive field S=9": lambda: fwd(lift_desc(S=9)),
        "nz=2": lambda: fwd(lift_desc(nz=2)),
        "frame range outside": lambda: fwd(lift_desc(f_begin=2, f_count=2), out_layout=1),
        "frame mode writes no ranks_out": lambda: fwd(lift_desc(f_begin=1, f_count=1), ranks_out=FAKE, out_layout=1),
        "frame mode writes fp32 channels-last": lambda: fwd(lift_desc(f_begin=1, f_count=1), out_layout=0),
        "peer outputs need frame mode": lambda: fwd(lift_desc(), out_layout=1, n_peers=1),
    }
    for msg, call in cases.items():
        assert call() == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())
    desc = lift_desc(cam_M=None)
    assert fwd(desc) == -1 and b"stp3_lift_splat_fwd_det: null pointer" in L.stp3_last_error()
    # the default query is not enough for the fixed-point grid (STP3_ENOSPC)
    small = L.stp3_lift_splat_workspace_bytes(lift_desc())
    assert fwd(lift_desc(), ws_bytes=small) != 0 and b"workspace too small" in L.stp3_last_error()


def test_spatial_sum_det_refusals_and_scratch():
    L = _lib.lib()
    assert L.stp3_spatial_sum_det_scratch_bytes(6, 2500, 64) == 6 * 128 * 2 * 64 * 8
    assert L.stp3_spatial_sum_det_scratch_bytes(2, 37, 1024) == 2 * 37 * 2 * 1024 * 8
    assert L.stp3_spatial_sum_det_scratch_bytes(2, 0, 64) == 0
    n = 1 << 30
    cases = {
        "bad argument": lambda: L.stp3_spatial_sum_det(FAKE, FAKE, 2, 16, 1025, FAKE, FAKE, n, None),
        "more than 65535 images": lambda: L.stp3_spatial_sum_det(FAKE, FAKE, 65536, 16, 64, FAKE, FAKE, n, None),
        "scratch smaller": lambda: L.stp3_spatial_sum_det(FAKE, FAKE, 2, 16, 64, FAKE, FAKE, 16, None),
    }
    for msg, call in cases.items():
        assert call() == -1, msg
        assert msg.encode() in L.stp3_last_error(), (msg, L.stp3_last_error())
    assert L.stp3_spatial_sum_det(None, FAKE, 2, 16, 64, FAKE, FAKE, n, None) == -1
