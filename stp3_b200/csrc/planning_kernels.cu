// Eval-mode planning (stp3/models/planning_model.py, stp3/cost.py): three launches per call.
//   plan_maps_kernel    one thread per (sample, cell): drivable probability, dangerous area and the lane-divider cost
//   plan_cost_kernel    one warp per (sample, candidate, frame): the footprint sums and Cost_Function.forward's terms
//   plan_refine_kernel  one CTA per sample: argmin over the command window, then the GRUCell / MLP refinement
// Every trajectory-derived index uses the reference's fp32 expressions with explicitly rounded operations (no FMA
// contraction, IEEE division), so each (row, column) the reference samples is the one sampled here.  Footprint sums are
// integer counts, except the headway sum, which each lane accumulates in a fixed order before a fixed shuffle tree.
// Nothing is accumulated with atomics and nothing is read back to the host.
#include <cstdint>

#include "common.cuh"

namespace stp3 {
namespace {

constexpr int kMaxT = 16;
constexpr int kMaxG = 512;
constexpr int kTile = 16;        // plan_maps_kernel: 16 x 16 cells per CTA
constexpr int kMaxLaneR = 8;     // lane-distance window radius the staged tile holds
constexpr int kMaxFootprint = 1 << 16;

struct Desc {
  int B, N, T, H, W;
  float dx0, dx1, bx0, bx1;
  int fp0[4], fp1[4];
  float safety, headway, lrdivider, comfort, progress, volume, rule, w0, w1, headway_dist, lane_dist;
  int n_hd, traj_c, G, lane_r;
};

// radius of the window that holds every lane cell within lane_dist of a cell: cells further out along either axis are
// at least (floor(L / dx) + 1) * dx > L away
inline int lane_radius(const stp3_plan_desc* d) {
  const float dmin = d->dx[0] < d->dx[1] ? d->dx[0] : d->dx[1];
  return (int)floorf(d->lane_dist / dmin) + 1;
}

// softmax over two logits, channel 1, as torch computes it: exp(l - max) / sum
__device__ __forceinline__ float softmax1(float l0, float l1) {
  const float m = fmaxf(l0, l1);
  const float e0 = expf(__fsub_rn(l0, m)), e1 = expf(__fsub_rn(l1, m));
  return __fdiv_rn(e1, __fadd_rn(e0, e1));
}

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }

// Tensor.long() (truncation toward zero) of fl(v + off), then clamp(., 0, n - 1)
__device__ __forceinline__ int cell_index(float v, float off, int n) {
  long long i = __float2ll_rz(__fadd_rn(v, off));
  i = i < 0 ? 0 : i;
  return (int)(i > n - 1 ? n - 1 : i);
}

__device__ __forceinline__ float sq(float v) { return __fmul_rn(v, v); }

__global__ void __launch_bounds__(kTile * kTile)
plan_maps_kernel(Desc d, const float* __restrict__ lane, const float* __restrict__ drivable, float* __restrict__ drv_map,
                 uint8_t* __restrict__ dang_map, float* __restrict__ lane_cost) {
  __shared__ uint8_t is_lane[(kTile + 2 * kMaxLaneR) * (kTile + 2 * kMaxLaneR)];
  const int b = blockIdx.z, R = d.lane_r, tw = kTile + 2 * R;
  const int r0 = blockIdx.y * kTile, c0 = blockIdx.x * kTile;
  const long long HW = (long long)d.H * d.W;
  const float* L = lane + (long long)b * d.n_hd * HW;
  for (int i = threadIdx.x; i < tw * tw; i += blockDim.x) {
    const int r = r0 - R + i / tw, c = c0 - R + i % tw;
    uint8_t v = 0;
    if (r >= 0 && r < d.H && c >= 0 && c < d.W) {
      const long long p = (long long)r * d.W + c;
      // cost.py:276-281: the lane probability is zeroed where <= 0.5, and torch.nonzero keeps what is left
      v = d.n_hd == 2 ? (softmax1(L[p], L[HW + p]) > 0.5f) : (L[p] != 0.f);
    }
    is_lane[i] = v;
  }
  __syncthreads();
  const int ty = threadIdx.x / kTile, tx = threadIdx.x % kTile;
  const int r = r0 + ty, c = c0 + tx;
  if (r >= d.H || c >= d.W) return;
  const long long p = (long long)r * d.W + c;
  const float* D = drivable + (long long)b * d.n_hd * HW;
  float drv;
  if (d.n_hd == 2) {
    drv = softmax1(D[p], D[HW + p]);
    if (drv < 0.5f) drv = 0.f;                     // cost.py:186-188 (< here, <= for the lane)
  } else {
    drv = D[p];
  }
  drv_map[b * HW + p] = drv;
  dang_map[b * HW + p] = drv == 0.f;               // torch.logical_not(drivable_area)
  // LR_divider (cost.py:290-298): sqrt((dr * dx[1])^2 + (dc * dx[0])^2) to every lane cell, the minimum
  float dist = INFINITY;
  for (int dr = -R; dr <= R; ++dr)
    for (int dc = -R; dc <= R; ++dc)
      if (is_lane[(ty + R + dr) * tw + tx + R + dc]) {
        const float e = __fsqrt_rn(__fadd_rn(sq(__fmul_rn((float)dr, d.dx1)), sq(__fmul_rn((float)dc, d.dx0))));
        dist = fminf(dist, e);
      }
  lane_cost[b * HW + p] = dist <= d.lane_dist ? __fmul_rn(sq(__fsub_rn(d.lane_dist, dist)), d.lrdivider) : 0.f;
}

// Sum over the warp in a fixed butterfly order
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Comfort + Progress of one candidate (cost.py:317-392) from its T points P (x flipped here); `use_target` is
// target_points.sum() >= 0.5 over the whole batch.  One pass over the frames, carrying the previous velocities.
__device__ float cost_fc_of(const Desc& d, const float* P, const float* tp, bool use_target) {
  const int T = d.T;
  float xp = 0.f, yp = 0.f, lat_vp = 0.f, lon_vp = 0.f, vp = 0.f, acc_p = 0.f;
  float lat_a = 0.f, lon_a = 0.f, jerk = 0.f, ymax = 0.f;
  for (int i = 0; i < T; ++i) {
    const float x = -P[i * d.traj_c], y = P[i * d.traj_c + 1];
    const float ddx = i == 0 ? x : __fsub_rn(x, xp);
    const float ddy = i == 0 ? y : __fsub_rn(y, yp);
    const float lat_v = __fdiv_rn(ddx, 0.5f), lon_v = __fdiv_rn(ddy, 0.5f);
    const float v = __fdiv_rn(__fsqrt_rn(__fadd_rn(sq(ddx), sq(ddy))), 0.5f);
    if (i >= 1) {
      lat_a = fmaxf(lat_a, fabsf(__fdiv_rn(__fsub_rn(lat_v, lat_vp), 0.5f)));
      lon_a = fmaxf(lon_a, fabsf(__fdiv_rn(__fsub_rn(lon_v, lon_vp), 0.5f)));
      const float acc = __fdiv_rn(__fsub_rn(v, vp), 0.5f);
      if (i >= 2) jerk = fmaxf(jerk, fabsf(__fdiv_rn(__fsub_rn(acc, acc_p), 0.5f)));
      acc_p = acc;
    }
    ymax = i == 0 ? y : fmaxf(ymax, y);
    xp = x; yp = y; lat_vp = lat_v; lon_vp = lon_v; vp = v;
  }
  float comfort = 0.f;
  comfort = __fadd_rn(comfort, sq(clampf(__fsub_rn(lat_a, 3.f), 0.f, 30.f)));
  comfort = __fadd_rn(comfort, sq(clampf(__fsub_rn(lon_a, 3.f), 0.f, 30.f)));
  comfort = __fadd_rn(comfort, sq(clampf(__fsub_rn(jerk, 1.f), 0.f, 20.f)));
  comfort = clampf(__fmul_rn(comfort, d.comfort), 0.f, 100.f);
  float far = 0.f;                    // the last point's squared distance to the target
  if (use_target) far = __fadd_rn(sq(__fsub_rn(xp, tp[0])), sq(__fsub_rn(yp, tp[1])));
  const float progress = clampf(__fmul_rn(__fsub_rn(far, ymax), d.progress), -100.f, 100.f);
  return __fadd_rn(comfort, progress);
}

__global__ void __launch_bounds__(256)
plan_cost_kernel(Desc d, const float* __restrict__ trajs, const uint8_t* __restrict__ occ, const float* __restrict__ cv,
                 const float* __restrict__ tp, const float* __restrict__ drv, const uint8_t* __restrict__ dang,
                 const float* __restrict__ lane_cost, float* __restrict__ cost_fc, float* __restrict__ cost_fo) {
  const long long warp = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (warp >= (long long)d.B * d.N * d.T) return;
  const int t = (int)(warp % d.T);
  const long long bn = warp / d.T;
  const int b = (int)(bn / d.N);
  const float* P = trajs + bn * d.T * d.traj_c;
  const float x = -P[t * d.traj_c], y = P[t * d.traj_c + 1];        // cost.py:34: x -> -x
  const long long HW = (long long)d.H * d.W;
  const uint8_t* O = occ + ((long long)b * d.T + t) * HW;
  const float* Dv = drv + b * HW;
  const uint8_t* Dg = dang + b * HW;

  // get_points (cost.py:92-100): rows from y / dx[1] + r, columns from x / dx[0] + c, each truncated and clamped
  const float yd = __fdiv_rn(y, d.dx1), xd = __fdiv_rn(x, d.dx0);
  const float yh = __fdiv_rn(__fadd_rn(y, d.headway_dist), d.dx1);   // HeadwayCost: y + L
  int n_occ0 = 0, n_dang = 0, n_occ1 = 0;
  float hw = 0.f;
  {
    const int nc = d.fp0[3] - d.fp0[2] + 1, n = (d.fp0[1] - d.fp0[0] + 1) * nc;
    for (int k = lane; k < n; k += 32) {
      const float rr = (float)(d.fp0[0] + k / nc), cc = (float)(d.fp0[2] + k % nc);
      const int col = cell_index(xd, cc, d.W);
      const long long p = (long long)cell_index(yd, rr, d.H) * d.W + col;
      n_occ0 += O[p];
      n_dang += Dg[p];
      const long long q = (long long)cell_index(yh, rr, d.H) * d.W + col;
      if (O[q]) hw = __fadd_rn(hw, Dv[q]);
    }
  }
  {
    const int nc = d.fp1[3] - d.fp1[2] + 1, n = (d.fp1[1] - d.fp1[0] + 1) * nc;
    for (int k = lane; k < n; k += 32) {
      const float rr = (float)(d.fp1[0] + k / nc), cc = (float)(d.fp1[2] + k % nc);
      n_occ1 += O[(long long)cell_index(yd, rr, d.H) * d.W + cell_index(xd, cc, d.W)];
    }
  }
  n_occ0 = __reduce_add_sync(0xffffffffu, n_occ0);
  n_dang = __reduce_add_sync(0xffffffffu, n_dang);
  n_occ1 = __reduce_add_sync(0xffffffffu, n_occ1);
  hw = warp_sum(hw);

  if (lane == 0) {
    // SafetyCost: o(0) * w[0] + o(lambda) * v * w[1], v the step length / 0.5 s
    const float px = t == 0 ? 0.f : -P[(t - 1) * d.traj_c], py = t == 0 ? 0.f : P[(t - 1) * d.traj_c + 1];
    const float ddx = t == 0 ? x : __fsub_rn(x, px), ddy = t == 0 ? y : __fsub_rn(y, py);
    const float vel = __fdiv_rn(__fsqrt_rn(__fadd_rn(sq(ddx), sq(ddy))), 0.5f);
    const float s = __fadd_rn(__fmul_rn((float)n_occ0, d.w0), __fmul_rn(__fmul_rn((float)n_occ1, vel), d.w1));
    const float safety = clampf(__fmul_rn(s, d.safety), 0.f, 100.f);
    const float headway = clampf(__fmul_rn(hw, d.headway), 0.f, 100.f);
    // discretize (cost.py:134-138): y with bx[0] / dx[0], x with bx[1] / dx[1]
    const int yi = cell_index(__fdiv_rn(__fsub_rn(y, d.bx0), d.dx0), 0.f, d.H);
    const int xi = cell_index(__fdiv_rn(__fsub_rn(x, d.bx1), d.dx1), 0.f, d.W);
    const long long pi = (long long)yi * d.W + xi;
    const float lr = clampf(lane_cost[b * HW + pi], 0.f, 100.f);
    const float vol = clampf(__fmul_rn(clampf(cv[((long long)b * d.T + t) * HW + pi], 0.f, 1000.f), d.volume), 0.f, 100.f);
    const float rule = clampf(__fmul_rn((float)n_dang, d.rule), 0.f, 100.f);
    cost_fo[warp] = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(safety, headway), lr), vol), rule);
    if (t == 0) {
      float s_tp = 0.f;                                             // target_points.sum(), in order
      for (int i = 0; i < 2 * d.B; ++i) s_tp = __fadd_rn(s_tp, tp[i]);
      cost_fc[bn] = cost_fc_of(d, P, tp + 2 * b, !(s_tp < 0.5f));
    }
  }
}

__device__ __forceinline__ float sigmoid_f(float v) { return 1.f / (1.f + expf(-v)); }

__global__ void __launch_bounds__(256)
plan_refine_kernel(Desc d, const int32_t* __restrict__ windows, const float* __restrict__ trajs,
                   const float* __restrict__ cost_fc, const float* __restrict__ cost_fo, const float* __restrict__ h0,
                   const float* __restrict__ tp, const float* __restrict__ w_ih, const float* __restrict__ b_ih,
                   const float* __restrict__ w_hh_t, const float* __restrict__ b_hh, const float* __restrict__ w1_t,
                   const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                   float* __restrict__ out_traj, int32_t* __restrict__ selected) {
  __shared__ float h[kMaxG], a[kMaxG], gi[3 * kMaxG], gh[3 * kMaxG];
  __shared__ float best_v[8];
  __shared__ int best_i[8];
  __shared__ float xin[6];
  const int b = blockIdx.x, tid = threadIdx.x, G = d.G, T = d.T;
  const int start = windows[2 * b], count = windows[2 * b + 1];

  // argmin of fc + sum_t fo over the window; lowest index on ties
  float bv = INFINITY;
  int bi = start;
  for (int n = start + tid; n < start + count; n += blockDim.x) {
    const long long bn = (long long)b * d.N + n;
    float s = 0.f;
    for (int t = 0; t < T; ++t) s = __fadd_rn(s, cost_fo[bn * T + t]);
    const float v = __fadd_rn(cost_fc[bn], s);
    if (v < bv) { bv = v; bi = n; }                  // n increases: the first minimum stays
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (tid % 32 == 0) { best_v[tid / 32] = bv; best_i[tid / 32] = bi; }
  for (int k = tid; k < G; k += blockDim.x) h[k] = h0[(long long)b * G + k];
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)blockDim.x / 32; ++w)
      if (best_v[w] < bv || (best_v[w] == bv && best_i[w] < bi)) { bv = best_v[w]; bi = best_i[w]; }
    best_i[0] = bi;
    selected[b] = bi;
    xin[0] = xin[1] = 0.f;
    xin[4] = tp[2 * b];
    xin[5] = tp[2 * b + 1];
  }
  __syncthreads();
  const float* sel = trajs + ((long long)b * d.N + best_i[0]) * T * d.traj_c;

  for (int t = 0; t < T; ++t) {
    if (tid == 0) {
      xin[2] = sel[t * d.traj_c];
      xin[3] = sel[t * d.traj_c + 1];
    }
    __syncthreads();
    // gate pre-activations: gi = W_ih x + b_ih, gh = W_hh h + b_hh (rows in gate order r, z, n)
    for (int j = tid; j < 3 * G; j += blockDim.x) {
      float s = b_ih[j];
#pragma unroll
      for (int k = 0; k < 6; ++k) s += w_ih[j * 6 + k] * xin[k];
      gi[j] = s;
      float u = b_hh[j];
      for (int k = 0; k < G; ++k) u += w_hh_t[(long long)k * 3 * G + j] * h[k];
      gh[j] = u;
    }
    __syncthreads();
    for (int j = tid; j < G; j += blockDim.x) {
      const float r = sigmoid_f(gi[j] + gh[j]);
      const float z = sigmoid_f(gi[G + j] + gh[G + j]);
      const float nn = tanhf(gi[2 * G + j] + r * gh[2 * G + j]);
      h[j] = (1.f - z) * nn + z * h[j];
    }
    __syncthreads();
    for (int j = tid; j < G; j += blockDim.x) {
      float s = b1[j];
      for (int k = 0; k < G; ++k) s += w1_t[(long long)k * G + j] * h[k];
      a[j] = fmaxf(s, 0.f);
    }
    __syncthreads();
    if (tid < 64) {                                   // warp 0: output x, warp 1: output y
      const int o = tid / 32, l = tid % 32;
      float s = 0.f;
      for (int k = l; k < G; k += 32) s += w2[o * G + k] * a[k];
      s = warp_sum(s) + b2[o];
      if (l == 0) {
        xin[o] = s;
        float* out = out_traj + ((long long)b * T + t) * 3;
        out[o] = s;
        if (o == 0) out[2] = 0.f;
      }
    }
    __syncthreads();
  }
}

Desc to_desc(const stp3_plan_desc* d) {
  Desc k;
  k.B = d->B; k.N = d->N; k.T = d->T; k.H = d->H; k.W = d->W;
  k.dx0 = d->dx[0]; k.dx1 = d->dx[1]; k.bx0 = d->bx[0]; k.bx1 = d->bx[1];
  for (int i = 0; i < 4; ++i) { k.fp0[i] = d->fp0[i]; k.fp1[i] = d->fp1[i]; }
  k.safety = d->safety; k.headway = d->headway; k.lrdivider = d->lrdivider; k.comfort = d->comfort;
  k.progress = d->progress; k.volume = d->volume; k.rule = d->rule; k.w0 = d->safety_w[0]; k.w1 = d->safety_w[1];
  k.headway_dist = d->headway_dist; k.lane_dist = d->lane_dist;
  k.n_hd = d->n_hd; k.traj_c = d->traj_c; k.G = d->G; k.lane_r = lane_radius(d);
  return k;
}

int check_footprint(const char* fn, const char* name, const int f[4]) {
  STP3_CHECK_ARG(f[0] >= 0 && f[2] >= 0 && f[0] <= f[1] && f[2] <= f[3], "%s: footprint %s [%d, %d] x [%d, %d] is empty "
                 "or has negative cells", fn, name, f[0], f[1], f[2], f[3]);
  STP3_CHECK_ARG((long long)(f[1] - f[0] + 1) * (f[3] - f[2] + 1) <= kMaxFootprint && f[1] < (1 << 20) &&
                 f[3] < (1 << 20), "%s: footprint %s is larger than %d cells", fn, name, kMaxFootprint);
  return STP3_OK;
}

// The descriptor's rules every entry point shares
int check_desc(const char* fn, const stp3_plan_desc* d) {
  STP3_CHECK_ARG(d != nullptr, "%s: desc is null", fn);
  STP3_CHECK_ARG(d->B > 0 && d->N > 0 && d->T > 0, "%s: B, N and T must be positive (got %d, %d, %d)", fn, d->B, d->N,
                 d->T);
  STP3_CHECK_ARG(d->T <= kMaxT, "%s: T = %d future frames, at most %d", fn, d->T, kMaxT);
  STP3_CHECK_ARG(d->N % 3 == 0, "%s: N = %d is not divisible by 3 (one third per command)", fn, d->N);
  STP3_CHECK_ARG(d->H > 0 && d->W > 0, "%s: bad grid %d x %d", fn, d->H, d->W);
  STP3_CHECK_ARG(d->H == d->W, "%s: non-square grid %d x %d (the reference's Rule and HeadwayCost reinterpret the map "
                 "as W x H)", fn, d->H, d->W);
  STP3_CHECK_ARG(d->dx[0] > 0.f && d->dx[1] > 0.f, "%s: dx must be positive", fn);
  STP3_CHECK_ARG(d->lane_dist >= 0.f && lane_radius(d) <= kMaxLaneR, "%s: the lane distance %g spans more than %d cells",
                 fn, d->lane_dist, kMaxLaneR);
  STP3_CHECK_ARG(d->n_hd == 1 || d->n_hd == 2, "%s: n_hd = %d, the hd map has 1 or 2 channels per element", fn, d->n_hd);
  STP3_CHECK_ARG(d->traj_c == 2 || d->traj_c == 3, "%s: traj_c = %d, points have 2 or 3 components", fn, d->traj_c);
  {
    const int rc0 = check_footprint(fn, "fp0", d->fp0);
    if (rc0 != STP3_OK) return rc0;
    const int rc1 = check_footprint(fn, "fp1", d->fp1);
    if (rc1 != STP3_OK) return rc1;
  }
  return STP3_OK;
}

}  // namespace
}  // namespace stp3

using namespace stp3;

extern "C" int stp3_plan_maps(const stp3_plan_desc* desc, const float* lane, const float* drivable, float* drv_map,
                              uint8_t* dang_map, float* lane_cost, void* stream) {
  const char* fn = "stp3_plan_maps";
  const int rc = check_desc(fn, desc);
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(lane && drivable && drv_map && dang_map && lane_cost, "%s: null pointer", fn);
  const Desc d = to_desc(desc);
  const dim3 grid((d.W + kTile - 1) / kTile, (d.H + kTile - 1) / kTile, d.B);
  plan_maps_kernel<<<grid, kTile * kTile, 0, static_cast<cudaStream_t>(stream)>>>(d, lane, drivable, drv_map, dang_map,
                                                                                   lane_cost);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_plan_cost(const stp3_plan_desc* desc, const float* trajs, const uint8_t* occupancy,
                              const float* cost_volume, const float* target_points, const float* drv_map,
                              const uint8_t* dang_map, const float* lane_cost, float* cost_fc, float* cost_fo,
                              void* stream) {
  const char* fn = "stp3_plan_cost";
  const int rc = check_desc(fn, desc);
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(trajs && occupancy && cost_volume && target_points && drv_map && dang_map && lane_cost && cost_fc &&
                 cost_fo, "%s: null pointer", fn);
  const Desc d = to_desc(desc);
  const long long warps = (long long)d.B * d.N * d.T;
  STP3_CHECK_ARG(warps <= (1LL << 34), "%s: too many (sample, candidate, frame) items", fn);
  plan_cost_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      d, trajs, occupancy, cost_volume, target_points, drv_map, dang_map, lane_cost, cost_fc, cost_fo);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_plan_refine(const stp3_plan_desc* desc, const int32_t* windows_host, const int32_t* windows,
                                const float* trajs, const float* cost_fc, const float* cost_fo, const float* h0,
                                const float* target_points, const float* w_ih, const float* b_ih, const float* w_hh_t,
                                const float* b_hh, const float* w1_t, const float* b1, const float* w2, const float* b2,
                                float* out_traj, int32_t* selected, void* stream) {
  const char* fn = "stp3_plan_refine";
  const int rc = check_desc(fn, desc);
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(windows_host && windows && trajs && cost_fc && cost_fo && h0 && target_points && w_ih && b_ih &&
                 w_hh_t && b_hh && w1_t && b1 && w2 && b2 && out_traj && selected, "%s: null pointer", fn);
  STP3_CHECK_ARG(desc->G > 0 && desc->G % 32 == 0 && desc->G <= kMaxG, "%s: G = %d must be a multiple of 32 in "
                 "[32, %d]", fn, desc->G, kMaxG);
  for (int b = 0; b < desc->B; ++b) {
    const int s = windows_host[2 * b], c = windows_host[2 * b + 1];
    STP3_CHECK_ARG(s >= 0 && c > 0 && (long long)s + c <= desc->N, "%s: window (%d, %d) of sample %d is outside "
                   "[0, %d)", fn, s, c, b, desc->N);
  }
  const Desc d = to_desc(desc);
  plan_refine_kernel<<<d.B, 256, 0, static_cast<cudaStream_t>(stream)>>>(d, windows, trajs, cost_fc, cost_fo, h0,
                                                                          target_points, w_ih, b_ih, w_hh_t, b_hh,
                                                                          w1_t, b1, w2, b2, out_traj, selected);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
