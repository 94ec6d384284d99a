// Fused lift-splat for sm_90a.  This file is compiled with ptxas -O1 (csrc/Makefile): the -O2/-O3 code ptxas 12.9 emits
// for lift_splat_scatter_tma_kernel faults with an illegal address in its pooling phase on the H100, while the same
// source at -O1 / -O0 runs clean and bit-exact (DESIGN.md §3.1).
//
//   K1  lift_splat_scatter_kernel : one CTA per (b, t, camera, tile of TW image columns)
//         phase A  depth logits and context features of the tile -> shared memory (coalesced tile loads),
//                  softmax over D in place (probabilities never leave the SM; the 371 MB/sample outer product of
//                  the reference, stp3.py:216, is never materialised)
//         phase B  frustum point -> ego frame -> sequential ego-motion warp -> voxel rank, with the reference's
//                  exact fp32 operation order (no FMA, IEEE division, truncation); rank staged beside the prob
//         phase C  outer product + pooling: a warp owns one image column; lanes own channel pairs and keep the
//                  column's context features in registers; walking the column for every depth bin is a segmented
//                  reduction over equal pillar ranks (all rows of a level camera fall into the same pillar),
//                  flushed with one coalesced red.global.add.v2.f32 per lane per segment into a channels-last
//                  (b,t,pillar,C) fp32 grid, plus one byte in a per-pillar occupancy map
//   K2  bev_finalize_kernel : temporal discount recurrence out[t] = out[t-1]*discount + grid[t] and the
//         channels-last -> (C,X,Y) transpose (lane = pillar, so stores are coalesced rows with no smem staging).
//         Reads (and re-zeroes) only the occupied pillars, so the scatter grid is left clean for the next call
//         and never needs a memset.
//
// Reference semantics: stp3/models/stp3.py:186-301, stp3/utils/geometry.py:299-318.
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "lift_geom.cuh"
#include "ptx.cuh"

namespace stp3 {

constexpr int kMaxFrames = 8;      // receptive field S supported by the in-kernel pose chain
constexpr int kScatterThreads = 256;
constexpr int kHChunk = 32;        // image rows whose features a lane keeps in registers at once
constexpr int kCChunk = 64;        // channels staged in shared memory at once (2 per lane)

struct LiftSplatParams {
  const float* feat;
  const float* depth;
  const float* cam_M;
  const float* cam_t;
  const float* ego_R;
  const float* ego_t;
  const float* xs;
  const float* ys;
  const float* ds;
  float off[3];
  float res[3];
  float inv[3];     // exact 1/res when res is a power of two
  int inv_ok[3];
  int nx, ny, nz;
  int B, S, N, D, Hf, Wf, C;
  int feat_nhwc;
  int use_depth;
  int f_begin;   // first flat frame (b*S + t) processed by this launch; CTAs enumerate f_begin + [0, f_count)
  int TW;        // image columns per CTA
  int tiles_w;   // ceil(Wf / TW)
  int32_t* ranks_out;
  float* grid;          // (B,S,nx*ny*nz,C) fp32, all-zero on entry
  unsigned char* occ;   // (B,S,nx*ny*nz) bytes, all-zero on entry; set to 1 where the grid was written
  // fixed-point mode only (stp3_lift_splat_fwd_det), indexed by the frame's slot in this launch
  long long* qgrid;         // (B,S,nx*ny*nz,C) int64 multiples of 2^-k_f, all-zero on entry
  const unsigned* fmax;     // bits of m_f, the largest finite |feature| of the frame
  unsigned* poison;         // per-frame bitmap of pillars that received a NaN or +-inf partial
  int lp;                   // ceil(log2(N * D * Hf * Wf)): points per frame
};

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// ---- 64-bit fixed point (deterministic mode).  A frame's partials are rounded to multiples of 2^-k_f with
// k_f = 62 - (ceil(log2 m_f) + ceil(log2 points)), so no pillar sum of the frame can reach 2^63 (every point adds at
// most m_f: probabilities are <= 1), and summed as int64: integer addition is associative, so the result does not
// depend on the order in which CTAs and warps arrive.
__host__ __device__ inline int ceil_log2_f32(unsigned bits) {   // bits of a finite float > 0
  const unsigned e = bits >> 23, m = bits & 0x7fffffu;
  if (e == 0) {                                                // subnormal m * 2^-149: -149 + ceil(log2 m)
    int c = 0;
    while ((1u << c) < m) ++c;
    return -149 + c;
  }
  return (int)e - 127 + (m != 0);
}

__host__ __device__ inline int frame_exponent(unsigned mbits, int lp) {
  return mbits == 0 ? 0 : 62 - (ceil_log2_f32(mbits) + lp);
}

// k_f of the frame in launch slot `slot`: the one place the kernels look up a frame's scale
__device__ __forceinline__ int slot_exponent(const unsigned* fmax, size_t slot, int lp) {
  return frame_exponent(fmax[slot], lp);
}

__device__ __forceinline__ double pow2d(int k) { return __hiloint2double((k + 1023) << 20, 0); }   // |k| <= 1022

__device__ __forceinline__ void red_add_u64(long long* addr, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

// where one frame's fixed-point partials go
struct FxSink {
  long long* grid;      // the frame's (pillar, C) int64 rows
  unsigned* poison;     // the frame's poison bitmap
  double scale;         // 2^k_f
};

__device__ __forceinline__ FxSink fx_sink(const LiftSplatParams& p, int bt, size_t nvox) {
  FxSink s;
  s.grid = p.qgrid + (size_t)bt * nvox * p.C;
  s.poison = p.poison + (size_t)bt * ((nvox + 31) / 32);
  s.scale = pow2d(slot_exponent(p.fmax, bt, p.lp));
  return s;
}

__device__ __forceinline__ void fx_add(const FxSink& s, int rank, long long* dst, float a) {
  if (isfinite(a)) {
    const long long q = __double2ll_rn((double)a * s.scale);
    if (q != 0) red_add_u64(dst, q);
  } else {
    atomicOr(s.poison + (rank >> 5), 1u << (rank & 31));
  }
}

// fixed-point counterpart of flush_segment
__device__ __forceinline__ void fx_flush(const FxSink& s, unsigned char* obase, int rank, int C, int c, bool mark,
                                         float a0, float a1) {
  if (c < C) {
    long long* dst = s.grid + (size_t)rank * C + c;
    fx_add(s, rank, dst, a0);
    if (c + 1 < C) fx_add(s, rank, dst + 1, a1);
  }
  if (mark) obase[rank] = 1;
}

// shared-memory row of channel (c0 + cl) in the feature tile: the two channels of a lane (2*lane, 2*lane+1) live in
// rows lane and lane+32, so that with an odd row stride the register fill of phase C is bank-conflict free
__device__ __forceinline__ int feat_row(int cl) { return ((cl & 1) << 5) | (cl >> 1); }

// flush one finished segment: lane owns channels (c, c+1) of pillar `rank`
__device__ __forceinline__ void flush_segment(float* gbase, unsigned char* obase, int rank, int C, int c, bool vec_ok,
                                              bool mark, float a0, float a1) {
  if (c < C) {
    float* dst = gbase + (size_t)rank * C + c;
    if (vec_ok) red_add_v2(dst, a0, a1);
    else { atomicAdd(dst, a0); if (c + 1 < C) atomicAdd(dst + 1, a1); }
  }
  if (mark) obase[rank] = 1;
}

// Tensor-core pooling (phase C of the TMA kernel).  For one image column the pooled rows of all depth bins are a small
// GEMM  out[d, c] = sum_h prob[d, h] * feat[h, c]  (M = D, K = Hf, N = C) whenever the points of a (depth, column) pair
// fall into one pillar -- every pair of a level camera, about half of them one degree off level.  It runs on the
// warp-level tensor-core path (mma.sync.m16n8k16, bf16 operands, fp32 accumulate) with both operands split into bf16
// hi + lo and the three products hi*hi + hi*lo + lo*hi, i.e. ~16 significand bits per operand like the hi/lo planes the
// BEV grid is stored in downstream.  A pair whose points fall into several pillars takes one more pass per pillar with
// the operand masked to it (up to kSegPasses); anything beyond that is left to a scalar segmented walk.
__device__ __forceinline__ void mma_bf16_m16n8k16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// TW = image columns per CTA (compile time so that tile indexing is shifts and immediates).
// Shared-memory tile layout (HP = Hf rounded up to 4 so that a column's probabilities are float4-readable):
//   s_prob [D][TW][HP] f32   softmax(depth) of the tile, zero in the padding rows
//   s_rank [D][TW][HP] i32   pillar rank or -1
//   s_col  [D][TW]     i32   rank shared by the whole image column (the usual case: a level camera maps a column
//                            of pixels at one depth into one pillar), -1 if the whole column is masked,
//                            -2 if the column spans several pillars (segmented slow path)
//   s_feat [64][npix|1] f32  context features of 64 channels, row permuted by feat_row()
// FX: fixed-point accumulation (see FxSink) instead of fp32 red.add.
template <int TW, bool FX>
__global__ void __launch_bounds__(kScatterThreads, 2)
lift_splat_scatter_kernel(const LiftSplatParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = p.D, Hf = p.Hf, Wf = p.Wf, C = p.C;
  const int HP = (Hf + 3) & ~3;
  const int npix = Hf * TW;
  const int fstride = (((Hf + kHChunk - 1) / kHChunk) * kHChunk * TW) | 1;   // odd, zero-padded to whole h-chunks
  float* s_prob = reinterpret_cast<float*>(smem_raw);
  int* s_rank = reinterpret_cast<int*>(s_prob + D * TW * HP);
  int* s_col = s_rank + D * TW * HP;
  float* s_feat = reinterpret_cast<float*>(s_col + D * TW);        // [kCChunk rows][fstride]
  float* s_mat = s_feat + kCChunk * fstride;                       // camera 12 + (kMaxFrames-1) * 12 pose floats
  float* s_ys = s_mat + 12 * kMaxFrames;                           // [Hf]
  float* s_ds = s_ys + Hf;                                         // [D]
  float* s_red = s_ds + D;                                         // [blockDim] softmax partials

  const int tid = threadIdx.x;
  const int nthr = blockDim.x;
  int blk = blockIdx.x;
  const int tile = blk % p.tiles_w; blk /= p.tiles_w;
  const int n = blk % p.N; blk /= p.N;
  const int frame = p.f_begin + blk;             // flat frame index b*S + t
  const int t = frame % p.S;
  const int b = frame / p.S;
  const int w0 = tile * TW;
  const int img = frame * p.N + n;               // camera-image index
  const int bt = blk;                            // slot of this frame in the scatter grid of this launch
  const int n_chain = p.S - 1 - t;               // poses t .. S-2 applied in order (stp3.py:270-277)

  // thread <-> pixel mapping shared by phases A and B: `parts` threads per pixel, each owning a slice of D
  const int npix_r = (npix + 31) & ~31;
  const int parts = max(1, nthr / npix_r);
  const int my_part = (nthr / npix_r) <= 1 ? 0 : tid / npix_r;
  const int dchunk = (D + parts - 1) / parts;

  // ---- small per-CTA constants
  if (tid < 9) s_mat[tid] = p.cam_M[img * 9 + tid];
  if (tid >= 9 && tid < 12) s_mat[tid] = p.cam_t[img * 3 + tid - 9];
  for (int i = tid; i < n_chain * 12; i += nthr) {
    const int k = i / 12, e = i % 12;
    const int src = b * p.S + t + k;
    s_mat[12 + i] = e < 9 ? p.ego_R[src * 9 + e] : p.ego_t[src * 3 + e - 9];
  }
  for (int i = tid; i < Hf; i += nthr) s_ys[i] = p.ys[i];
  for (int i = tid; i < D; i += nthr) s_ds[i] = p.ds[i];
  if (HP != Hf)                                                    // zero the padding rows once
    for (int i = tid; i < D * TW * (HP - Hf); i += nthr) {
      const int col = i / (HP - Hf), r = i % (HP - Hf);
      s_prob[col * HP + Hf + r] = 0.f;
      s_rank[col * HP + Hf + r] = -1;
    }
  __syncthreads();

  // ---- phases A + B, one pass over the pixels this thread owns
  const float offx = p.off[0], offy = p.off[1], offz = p.off[2];
  const float resx = p.res[0], resy = p.res[1], resz = p.res[2];
  const float fnx = (float)p.nx, fny = (float)p.ny, fnz = (float)p.nz;
  for (int px0 = 0; px0 < npix; px0 += (parts == 1 ? nthr : npix_r)) {
    const int px = px0 + (parts == 1 ? tid : tid % npix_r);
    const bool act = px < npix && my_part < parts;
    const int wl = px % TW, h = px / TW;
    const int w = w0 + wl;
    const bool inb = act && w < Wf;
    const int da = my_part * dchunk, db = act ? min(D, da + dchunk) : da;
    float* prow = s_prob + wl * HP + h;          // + d*TW*HP
    // A: logits -> smem, softmax over D (stp3.py:215)
    if (p.use_depth) {
      const float* dsrc = p.depth + ((size_t)img * D * Hf + h) * Wf + w;
      float mx = -INFINITY;
      for (int d = da; d < db; ++d) {
        const float v = inb ? __ldg(dsrc + (size_t)d * Hf * Wf) : 0.f;
        prow[d * TW * HP] = v;
        mx = fmaxf(mx, v);
      }
      if (parts > 1) {
        s_red[tid] = mx;
        __syncthreads();
        if (act) for (int q = 0; q < parts; ++q) mx = fmaxf(mx, s_red[q * npix_r + px - px0]);
        __syncthreads();
      }
      float sum = 0.f;
      for (int d = da; d < db; ++d) {
        const float e = __expf(prow[d * TW * HP] - mx);
        prow[d * TW * HP] = e;
        sum += e;
      }
      if (parts > 1) {
        s_red[tid] = sum;
        __syncthreads();
        sum = 0.f;
        if (act) for (int q = 0; q < parts; ++q) sum += s_red[q * npix_r + px - px0];
        __syncthreads();
      }
      const float inv = __frcp_rn(sum);
      for (int d = da; d < db; ++d) prow[d * TW * HP] *= inv;
    } else {
      for (int d = da; d < db; ++d) prow[d * TW * HP] = 1.0f;      // stp3.py:218
    }
    // B: voxel rank of every point of this pixel's ray (bit-exact with the reference CPU path)
    if (act) {
      int* rrow = s_rank + wl * HP + h;
      const float xw = inb ? __ldg(p.xs + w) : 0.f;
      const float yh = s_ys[h];
      for (int d = da; d < db; ++d) {
        int rank = -1;
        if (inb) {
          const float dep = s_ds[d];
          float x = __fmul_rn(xw, dep);                  // stp3.py:195: (u*d, v*d, d)
          float y = __fmul_rn(yh, dep);
          float z = dep;
          affine_exact(s_mat, s_mat + 9, x, y, z);       // stp3.py:196-198
          for (int k = 0; k < n_chain; ++k)              // stp3.py:270-277, sequential, rounded every step
            affine_exact(s_mat + 12 + 12 * k, s_mat + 12 + 12 * k + 9, x, y, z);
          // stp3.py:287-289: ((p - (start - res/2)) / res).long() -- true division, truncation toward zero;
          // trunc(q) in [0, n)  <=>  -1 < q < n  (keeps the (-1,0) band in cell 0 exactly like .long()).
          // (a power-of-two resolution makes the division an exact scaling: multiply by the exact reciprocal)
          const float qx = p.inv_ok[0] ? __fmul_rn(__fsub_rn(x, offx), p.inv[0]) : __fdiv_rn(__fsub_rn(x, offx), resx);
          const float qy = p.inv_ok[1] ? __fmul_rn(__fsub_rn(y, offy), p.inv[1]) : __fdiv_rn(__fsub_rn(y, offy), resy);
          const float qz = p.inv_ok[2] ? __fmul_rn(__fsub_rn(z, offz), p.inv[2]) : __fdiv_rn(__fsub_rn(z, offz), resz);
          const bool keep = (qx > -1.f) && (qx < fnx) && (qy > -1.f) && (qy < fny) && (qz > -1.f) && (qz < fnz);
          if (keep) {
            const int ix = (int)qx, iy = (int)qy, iz = (int)qz;     // cvt.rzi
            rank = ix * (p.ny * p.nz) + iy * p.nz + iz;              // stp3.py:251-255
          }
          if (p.ranks_out) p.ranks_out[(((size_t)img * D + d) * Hf + h) * Wf + w] = rank;
        }
        rrow[d * TW * HP] = rank;
        if (rank < 0) prow[d * TW * HP] = 0.f;     // masked points contribute nothing (stp3.py:239-248)
      }
    }
  }
  __syncthreads();
  // column summary: one thread per (d, wl)
  for (int i = tid; i < D * TW; i += nthr) {
    const int* r = s_rank + i * HP;
    int first = -1;
    bool uni = true;
    for (int h = 0; h < Hf; ++h) {
      const int v = r[h];
      if (v >= 0) { uni &= (first < 0 || v == first); first = v; }
    }
    s_col[i] = uni ? first : -2;                 // masked rows carry probability 0, so they never split a column
  }

  // ---- phase C: outer product + segmented pooling.  work item = (column, depth slice); lanes = channel pairs
  const int warp = tid >> 5, lane = tid & 31;
  const int nwarps = nthr >> 5;
  const int dsplit = max(1, nwarps / TW);
  const int dper = (D + dsplit - 1) / dsplit;
  const size_t nvox = (size_t)p.nx * p.ny * p.nz;
  float* gbase = p.grid + (size_t)bt * nvox * C;
  unsigned char* obase = p.occ + (size_t)bt * nvox;
  const bool vec_ok = (C % 2) == 0;
  FxSink fx;
  if constexpr (FX) fx = fx_sink(p, bt, nvox);
  for (int i = tid; i < kCChunk * (fstride - npix); i += nthr)     // zero padding of the feature rows (once)
    s_feat[(i / (fstride - npix)) * fstride + npix + i % (fstride - npix)] = 0.f;
  for (int c0 = 0; c0 < C; c0 += kCChunk) {
    // stage the context features of channels [c0, c0+64) of this tile (stp3.py:216 re-reads them D times)
    __syncthreads();
    if (p.feat_nhwc) {
      for (int px = tid / kCChunk; px < npix; px += nthr / kCChunk) {
        const int cl = tid % kCChunk;
        const int wl = px % TW, h = px / TW;
        const int w = w0 + wl, c = c0 + cl;
        float v = 0.f;
        if (w < Wf && c < C) v = __ldg(p.feat + (((size_t)img * Hf + h) * Wf + w) * C + c);
        s_feat[feat_row(cl) * fstride + px] = v;
      }
    } else {
      for (int px0 = 0; px0 < npix; px0 += npix_r) {
        const int px = px0 + tid % npix_r;
        if (px < npix && my_part < parts) {
          const int wl = px % TW, h = px / TW;
          const int w = w0 + wl;
          const float* src = p.feat + (((size_t)img * C + c0) * Hf + h) * Wf + w;
          for (int cl = my_part; cl < kCChunk; cl += parts) {
            float v = 0.f;
            if (w < Wf && c0 + cl < C) v = __ldg(src + (size_t)cl * Hf * Wf);
            s_feat[feat_row(cl) * fstride + px] = v;
          }
        }
      }
    }
    __syncthreads();
    const int c = c0 + 2 * lane;
    const bool mark = (lane == 0) && (c0 == 0);
    for (int item = warp; item < TW * dsplit; item += nwarps) {
      const int wl = item % TW;
      if (w0 + wl >= Wf) continue;
      const int d0 = (item / TW) * dper;
      const int d1 = min(D, d0 + dper);
      for (int h0 = 0; h0 < Hf; h0 += kHChunk) {
        float f0[kHChunk], f1[kHChunk];
#pragma unroll
        for (int j = 0; j < kHChunk; ++j) {          // rows >= Hf read the zero padding
          f0[j] = s_feat[lane * fstride + (h0 + j) * TW + wl];
          f1[j] = s_feat[(lane + 32) * fstride + (h0 + j) * TW + wl];
        }
        for (int d = d0; d < d1; ++d) {
          const int col = s_col[d * TW + wl];
          if (col == -1) continue;                   // the whole column is outside the grid
          const float* pr = s_prob + (d * TW + wl) * HP + h0;
          if (col >= 0) {
            // fast path: the column is one segment -> 8 FFMA per broadcast LDS.128, one flush
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int j4 = 0; j4 < kHChunk / 4; ++j4) {
              if (h0 + 4 * j4 < Hf) {
                const float4 q = *reinterpret_cast<const float4*>(pr + 4 * j4);
                a0 = fmaf(q.x, f0[4 * j4 + 0], a0); a1 = fmaf(q.x, f1[4 * j4 + 0], a1);
                a0 = fmaf(q.y, f0[4 * j4 + 1], a0); a1 = fmaf(q.y, f1[4 * j4 + 1], a1);
                a0 = fmaf(q.z, f0[4 * j4 + 2], a0); a1 = fmaf(q.z, f1[4 * j4 + 2], a1);
                a0 = fmaf(q.w, f0[4 * j4 + 3], a0); a1 = fmaf(q.w, f1[4 * j4 + 3], a1);
              }
            }
            if constexpr (FX) fx_flush(fx, obase, col, C, c, mark, a0, a1);
            else flush_segment(gbase, obase, col, C, c, vec_ok, mark, a0, a1);
          } else {
            // slow path: segmented reduction over equal ranks along the column
            const int* rk = s_rank + (d * TW + wl) * HP + h0;
            int cur = -1;
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int j = 0; j < kHChunk; ++j) {
              if (h0 + j < Hf) {
                const int r = rk[j];
                if (r != cur) {                      // warp-uniform: segment boundary
                  if (cur >= 0) {
                    if constexpr (FX) fx_flush(fx, obase, cur, C, c, mark, a0, a1);
                    else flush_segment(gbase, obase, cur, C, c, vec_ok, mark, a0, a1);
                  }
                  cur = r; a0 = 0.f; a1 = 0.f;
                }
                const float q = pr[j];
                a0 = fmaf(q, f0[j], a0);
                a1 = fmaf(q, f1[j], a1);
              }
            }
            if (cur >= 0) {
              if constexpr (FX) fx_flush(fx, obase, cur, C, c, mark, a0, a1);
              else flush_segment(gbase, obase, cur, C, c, vec_ok, mark, a0, a1);
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// TMA-staged variant (the fast path: 4-column tiles, Wf % 4 == 0).  Same phases and the same arithmetic as
// lift_splat_scatter_kernel, but the tile's depth logits and context features are fetched by the TMA unit
// (cp.async.bulk.tensor, 3-D boxes) the moment the CTA starts, and the pure-ALU rank computation (phase B) runs while
// they are in flight; nothing in the kernel waits on a global load except the two mbarrier waits.
//   logits   box (4 w, Hf, D)      -> s_stage [D][Hf][4]            (softmax transposes it into s_prob [D][4][HP])
//   features NHWC: 1 box (64 ch, 4 w, Hf)  -> s_feat[Hf][4][64]
//            NCHW: 1 box (4 w, Hf, 64 ch)  -> s_feat[64][Hf][4]   (only the mma B-fragment loads of phase C read it: 64 LDS
//                  per warp and column, so their bank conflicts do not matter)
constexpr int kTmaTW = 4;
constexpr int kSegPasses = 4;      // pillars per (depth bin, image column) pair the tensor-core passes cover

// Pillar ranks of the depth bins [da, db) of one pixel's ray, bit-exact with the reference (lift_geom.cuh).  NC ego-motion
// links (0, 1, 2) are compile-time and live in registers with the camera transform; NC = 3: two in registers, the rest of a
// longer chain walks the shared-memory copies.  POW2: x / y resolutions are powers of two and nz == 1 (lift_geom.cuh).
template <int NC, bool POW2>
__device__ __forceinline__ void ray_ranks(const BevQuant& q, const float* __restrict__ s_mat, const float* __restrict__ s_ds,
                                          int n_chain, int da, int db, float xw, float yh, int* __restrict__ rrow,
                                          int rstride, int32_t* __restrict__ rout, size_t ostride) {
  float cm[12], e0[12], e1[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    cm[i] = s_mat[i];
    e0[i] = NC > 0 ? s_mat[12 + i] : 0.f;
    e1[i] = NC > 1 ? s_mat[24 + i] : 0.f;
  }
  for (int d = da; d < db; ++d) {
    const float dep = s_ds[d];
    float x = __fmul_rn(xw, dep);                  // stp3.py:195: (u*d, v*d, d)
    float y = __fmul_rn(yh, dep);
    float z = dep;
    affine_exact(cm, cm + 9, x, y, z);             // stp3.py:196-198
    if (NC > 0) affine_exact(e0, e0 + 9, x, y, z); // stp3.py:270-277, sequential, rounded every step
    if (NC > 1) affine_exact(e1, e1 + 9, x, y, z);
    if (NC > 2)
      for (int k = 2; k < n_chain; ++k) affine_exact(s_mat + 12 + 12 * k, s_mat + 12 + 12 * k + 9, x, y, z);
    const int rank = POW2 ? quantise_rank_pow2xy_nz1(q, x, y, z) : quantise_rank(q, x, y, z);   // stp3.py:287-289, 239-255
    if (rout) rout[(size_t)d * ostride] = rank;
    rrow[d * rstride] = rank;
  }
}

struct LiftSplatTmaMaps {
  CUtensorMap depth;   // (Wf, Hf, D * n_img) fp32
  CUtensorMap feat;    // NCHW: (Wf, Hf, C * n_img) fp32 ; NHWC: (C, Wf, Hf * n_img) fp32
};

template <bool FX>
__global__ void __launch_bounds__(kScatterThreads, 2)
lift_splat_scatter_tma_kernel(const __grid_constant__ LiftSplatTmaMaps maps, const LiftSplatParams p) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem_raw = smem_dyn + ((128u - (ptx::smem_u32(smem_dyn) & 127u)) & 127u);
  constexpr int TW = kTmaTW;
  const int D = p.D, Hf = p.Hf, Wf = p.Wf, C = p.C;
  const int HP = (Hf + 3) & ~3;
  const int npix = Hf * TW;
  const int fstride = npix;                                        // NCHW tile: [64 channels][Hf][TW]
  const int feat_floats = npix * kCChunk;
  float* s_stage = reinterpret_cast<float*>(smem_raw);             // [D][Hf][TW] raw logits (TMA destination)
  float* s_feat = s_stage + ((D * npix + 31) & ~31);               // feature tile (TMA destination)
  float* s_prob = s_feat + ((feat_floats + 31) & ~31);             // [D][TW][HP]
  int* s_rank = reinterpret_cast<int*>(s_prob + D * TW * HP);      // [D][TW][HP]
  int* s_seg = s_rank + D * TW * HP;                               // [kSegPasses][D][TW] k-th distinct pillar of the (depth, column) pair, -1 = none
  int* s_nseg = s_seg + kSegPasses * D * TW;                       // [D][TW] distinct pillars: 0 .. kSegPasses, kSegPasses + 1 = more
  int* s_cinfo = s_nseg + D * TW;                                  // [TW] max of s_nseg over the column's depth bins
  float* s_mat = reinterpret_cast<float*>(s_cinfo + TW);           // camera 12 + (kMaxFrames-1) * 12 pose floats
  float* s_ys = s_mat + 12 * kMaxFrames;
  float* s_ds = s_ys + Hf;
  float* s_red = s_ds + D;                                         // [blockDim]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_red + kScatterThreads + (((Hf + D) & 1) ? 1 : 0));

  const int tid = threadIdx.x;
  const int nthr = blockDim.x;
  int blk = blockIdx.x;
  const int tile = blk % p.tiles_w; blk /= p.tiles_w;
  const int n = blk % p.N; blk /= p.N;
  const int frame = p.f_begin + blk;
  const int t = frame % p.S;
  const int b = frame / p.S;
  const int w0 = tile * TW;
  const int img = frame * p.N + n;
  const int bt = blk;
  const int n_chain = p.S - 1 - t;

  if (tid == 0) {
    ptx::mbar_init(&bars[0], 1);
    ptx::mbar_init(&bars[1], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int npix_r = (npix + 31) & ~31;
  const int parts = max(1, nthr / npix_r);
  const int my_part = (nthr / npix_r) <= 1 ? 0 : tid / npix_r;
  const int dchunk = (D + parts - 1) / parts;

  // start the feature tile of channels [c0, c0+64): one TMA box, issued by thread 0
  auto issue_features = [&](int c0) {
    if (tid == 0) {
      ptx::mbar_arrive_expect_tx(&bars[1], (uint32_t)(npix * kCChunk * 4));
      if (p.feat_nhwc) ptx::tma_load_3d(s_feat, &maps.feat, &bars[1], c0, w0, img * Hf);
      else ptx::tma_load_3d(s_feat, &maps.feat, &bars[1], w0, 0, img * C + c0);
    }
  };
  if (tid == 0 && p.use_depth) {
    ptx::mbar_arrive_expect_tx(&bars[0], (uint32_t)(D * npix * 4));
    ptx::tma_load_3d(s_stage, &maps.depth, &bars[0], w0, 0, img * D);
  }
  issue_features(0);

  if (tid < 9) s_mat[tid] = p.cam_M[img * 9 + tid];
  if (tid >= 9 && tid < 12) s_mat[tid] = p.cam_t[img * 3 + tid - 9];
  for (int i = tid; i < n_chain * 12; i += nthr) {
    const int k = i / 12, e = i % 12;
    const int src = b * p.S + t + k;
    s_mat[12 + i] = e < 9 ? p.ego_R[src * 9 + e] : p.ego_t[src * 3 + e - 9];
  }
  for (int i = tid; i < Hf; i += nthr) s_ys[i] = p.ys[i];
  for (int i = tid; i < D; i += nthr) s_ds[i] = p.ds[i];
  if (HP != Hf)
    for (int i = tid; i < D * TW * (HP - Hf); i += nthr) {
      const int col = i / (HP - Hf), r = i % (HP - Hf);
      s_prob[col * HP + Hf + r] = 0.f;
      s_rank[col * HP + Hf + r] = -1;
    }
  __syncthreads();

  // ---- phase B (pure ALU, overlaps the TMA transfers): voxel rank of every point, bit-exact with the reference
  BevQuant bq;
#pragma unroll
  for (int i = 0; i < 3; ++i) { bq.off[i] = p.off[i]; bq.res[i] = p.res[i]; bq.inv[i] = p.inv[i]; bq.inv_ok[i] = p.inv_ok[i]; }
  bq.nx = p.nx; bq.ny = p.ny; bq.nz = p.nz;
  const bool pow2 = p.inv_ok[0] && p.inv_ok[1] && p.nz == 1 && p.res[2] > 0.f;
  for (int px0 = 0; px0 < npix; px0 += (parts == 1 ? nthr : npix_r)) {
    const int px = px0 + (parts == 1 ? tid : tid % npix_r);
    const bool act = px < npix && my_part < parts;
    if (!act) continue;
    const int wl = px % TW, h = px / TW;
    const int w = w0 + wl;
    const bool inb = w < Wf;
    const int da = my_part * dchunk, db = min(D, da + dchunk);
    int* rrow = s_rank + wl * HP + h;
    const float xw = inb ? __ldg(p.xs + w) : 0.f;
    const float yh = s_ys[h];
    int32_t* rout = p.ranks_out ? p.ranks_out + ((size_t)img * D * Hf + h) * Wf + w : nullptr;
    if (!inb) {
      for (int d = da; d < db; ++d) rrow[d * TW * HP] = -1;
      continue;
    }
    const size_t ost = (size_t)Hf * Wf;
#define STP3_RAY(NC_)                                                                                             \
    do {                                                                                                          \
      if (pow2) ray_ranks<NC_, true>(bq, s_mat, s_ds, n_chain, da, db, xw, yh, rrow, TW * HP, rout, ost);            \
      else ray_ranks<NC_, false>(bq, s_mat, s_ds, n_chain, da, db, xw, yh, rrow, TW * HP, rout, ost);                \
    } while (0)
    if (n_chain == 0) STP3_RAY(0);
    else if (n_chain == 1) STP3_RAY(1);
    else if (n_chain == 2) STP3_RAY(2);
    else STP3_RAY(3);
#undef STP3_RAY
  }
  __syncthreads();

  // ---- phase A: softmax over D of the TMA-landed logits, written transposed ([d][wl][h]) with masked points zeroed
  if (p.use_depth) ptx::mbar_wait(&bars[0], 0);
  for (int px0 = 0; px0 < npix; px0 += (parts == 1 ? nthr : npix_r)) {
    const int px = px0 + (parts == 1 ? tid : tid % npix_r);
    const bool act = px < npix && my_part < parts;
    const int wl = px % TW, h = px / TW;
    const int da = my_part * dchunk, db = act ? min(D, da + dchunk) : da;
    const float* srow = s_stage + px;               // + d*npix   ([d][h][w], px = h*TW + wl)
    float* prow = s_prob + wl * HP + h;             // + d*TW*HP
    const int* rrow = s_rank + wl * HP + h;
    if (p.use_depth) {
      float mx = -INFINITY;
      for (int d = da; d < db; ++d) mx = fmaxf(mx, srow[d * npix]);
      if (parts > 1) {
        s_red[tid] = mx;
        __syncthreads();
        if (act) for (int q = 0; q < parts; ++q) mx = fmaxf(mx, s_red[q * npix_r + px - px0]);
        __syncthreads();
      }
      float sum = 0.f;
      for (int d = da; d < db; ++d) {
        const float e = __expf(srow[d * npix] - mx);
        prow[d * TW * HP] = e;
        sum += e;
      }
      if (parts > 1) {
        s_red[tid] = sum;
        __syncthreads();
        sum = 0.f;
        if (act) for (int q = 0; q < parts; ++q) sum += s_red[q * npix_r + px - px0];
        __syncthreads();
      }
      const float inv = __frcp_rn(sum);
      for (int d = da; d < db; ++d) prow[d * TW * HP] = rrow[d * TW * HP] < 0 ? 0.f : prow[d * TW * HP] * inv;
    } else {
      for (int d = da; d < db; ++d) prow[d * TW * HP] = rrow[d * TW * HP] < 0 ? 0.f : 1.0f;
    }
  }
  __syncthreads();
  if (tid < TW) s_cinfo[tid] = 0;
  __syncthreads();
  for (int i = tid; i < D * TW; i += nthr) {       // summary of every (depth, column) pair: its first kSegPasses pillars
    const int* r = s_rank + i * HP;
    int rs[kSegPasses];
#pragma unroll
    for (int k = 0; k < kSegPasses; ++k) rs[k] = -1;
    int n = 0;
    for (int h = 0; h < Hf; ++h) {
      const int v = r[h];
      bool seen = v < 0;                           // masked rows carry probability 0: they never split a pair
#pragma unroll
      for (int k = 0; k < kSegPasses; ++k) seen |= (v == rs[k]);
      if (!seen) {
#pragma unroll
        for (int k = 0; k < kSegPasses; ++k) if (k == n) rs[k] = v;
        n = min(n + 1, kSegPasses + 1);
      }
    }
#pragma unroll
    for (int k = 0; k < kSegPasses; ++k) s_seg[k * D * TW + i] = rs[k];
    s_nseg[i] = n;
    if (n > 0) atomicMax(&s_cinfo[i % TW], n);
  }
  __syncthreads();

  // ---- phase C: pooling on the tensor cores (ptx::split_hilo, mma_bf16_m16n8k16 below).
  // warp = (image column wl, half of the 64 channels); per m-tile of 16 depth bins: A = probabilities masked to the
  // pass's pillar (16 x Hf), B = the column's features (Hf x 32 channels, fragments loaded once per channel chunk),
  // accumulators flushed with one red.global.add.v2.f32 per lane and (depth bin, 8-channel group).
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, tg = lane & 3;
  const int wl = warp & (TW - 1), nhalf = warp / TW;            // 8 warps: 4 columns x 2 channel halves
  const size_t nvox = (size_t)p.nx * p.ny * p.nz;
  float* gbase = p.grid + (size_t)bt * nvox * C;
  unsigned char* obase = p.occ + (size_t)bt * nvox;
  FxSink fx;
  if constexpr (FX) fx = fx_sink(p, bt, nvox);
  constexpr int KS = 2;                                         // k-steps of 16 image rows: Hf <= 32 (host-checked)
  const int n_mt = (D + 15) >> 4;
  const bool col_ok = w0 + wl < Wf;
  const int cmax = s_cinfo[wl];                                  // 0: nothing of this column lands in the grid
  uint32_t fphase = 0;
  for (int c0 = 0; c0 < C; c0 += kCChunk) {
    ptx::mbar_wait(&bars[1], fphase);
    fphase ^= 1;
    if (col_ok && cmax > 0) {
      // B fragments: b0 = (k = 2tg, 2tg+1; n = g), b1 = (k = 2tg+8, 2tg+9; n = g) of every 16 x 8 block
      uint32_t bh[4][KS][2], bl[4][KS][2];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int cl = nhalf * 32 + nt * 8 + g;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int h = ks * 16 + r * 8 + 2 * tg;
            float x0 = 0.f, x1 = 0.f;
            if (p.feat_nhwc) {
              if (h < Hf) x0 = s_feat[(h * TW + wl) * kCChunk + cl];
              if (h + 1 < Hf) x1 = s_feat[((h + 1) * TW + wl) * kCChunk + cl];
            } else {
              if (h < Hf) x0 = s_feat[cl * fstride + h * TW + wl];
              if (h + 1 < Hf) x1 = s_feat[cl * fstride + (h + 1) * TW + wl];
            }
            ptx::split_hilo(x0, x1, bh[nt][ks][r], bl[nt][ks][r]);
          }
        }
      }
      const int n_pass = min(cmax, kSegPasses);
      for (int pass = 0; pass < n_pass; ++pass) {
        const int* seg = s_seg + pass * D * TW;
        for (int mt = 0; mt < n_mt; ++mt) {
          const int d_lo = mt * 16 + g, d_hi = d_lo + 8;
          const int seg_lo = d_lo < D ? seg[d_lo * TW + wl] : -1;
          const int seg_hi = d_hi < D ? seg[d_hi * TW + wl] : -1;
          if (__ballot_sync(0xffffffffu, (seg_lo >= 0) || (seg_hi >= 0)) == 0u) continue;
          // A fragments: a0 = (row g, k = 2tg, 2tg+1), a1 = (row g+8, same k), a2 / a3 = the same rows at k + 8
          uint32_t ah[KS][4], al[KS][4];
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              const int h = ks * 16 + (r >> 1) * 8 + 2 * tg;
              const int sg = (r & 1) ? seg_hi : seg_lo;
              const int d = (r & 1) ? d_hi : d_lo;
              float x0 = 0.f, x1 = 0.f;
              if (sg >= 0 && h < HP) {
                const float2 q = *reinterpret_cast<const float2*>(s_prob + (d * TW + wl) * HP + h);
                const int2 rk = *reinterpret_cast<const int2*>(s_rank + (d * TW + wl) * HP + h);
                x0 = rk.x == sg ? q.x : 0.f;
                x1 = rk.y == sg ? q.y : 0.f;
              }
              ptx::split_hilo(x0, x1, ah[ks][r], al[ks][r]);
            }
          }
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
              mma_bf16_m16n8k16(acc, ah[ks], bh[nt][ks][0], bh[nt][ks][1]);
              mma_bf16_m16n8k16(acc, ah[ks], bl[nt][ks][0], bl[nt][ks][1]);
              mma_bf16_m16n8k16(acc, al[ks], bh[nt][ks][0], bh[nt][ks][1]);
            }
            // c0, c1 = (row g, columns 2tg, 2tg+1); c2, c3 = (row g+8, same columns)
            const int c = c0 + nhalf * 32 + nt * 8 + 2 * tg;
            if constexpr (FX) {
              if (seg_lo >= 0) {
                fx_add(fx, seg_lo, fx.grid + (size_t)seg_lo * C + c, acc[0]);
                fx_add(fx, seg_lo, fx.grid + (size_t)seg_lo * C + c + 1, acc[1]);
              }
              if (seg_hi >= 0) {
                fx_add(fx, seg_hi, fx.grid + (size_t)seg_hi * C + c, acc[2]);
                fx_add(fx, seg_hi, fx.grid + (size_t)seg_hi * C + c + 1, acc[3]);
              }
            } else {
              if (seg_lo >= 0) red_add_v2(gbase + (size_t)seg_lo * C + c, acc[0], acc[1]);
              if (seg_hi >= 0) red_add_v2(gbase + (size_t)seg_hi * C + c, acc[2], acc[3]);
            }
          }
          if (c0 == 0 && nhalf == 0 && tg == 0) {
            if (seg_lo >= 0) obase[seg_lo] = 1;
            if (seg_hi >= 0) obase[seg_hi] = 1;
          }
        }
      }
      // leftovers: (depth, column) pairs that touch more than kSegPasses pillars -- segmented walk over the rows that
      // belong to none of the pillars the tensor-core passes covered; lanes own channel pairs, the two warps of the
      // column split the depth bins
      if (cmax > kSegPasses) {
        const int c = c0 + 2 * lane;
        for (int d = nhalf; d < D; d += 2) {
          if (s_nseg[d * TW + wl] <= kSegPasses) continue;
          int ex[kSegPasses];
#pragma unroll
          for (int k = 0; k < kSegPasses; ++k) ex[k] = s_seg[k * D * TW + d * TW + wl];
          const int* rk = s_rank + (d * TW + wl) * HP;
          const float* pr = s_prob + (d * TW + wl) * HP;
          int cur = -1;
          float a0 = 0.f, a1 = 0.f;
          for (int h = 0; h < Hf; ++h) {
            const int r = rk[h];
            bool skip = r < 0;
#pragma unroll
            for (int k = 0; k < kSegPasses; ++k) skip |= (r == ex[k]);
            if (skip) continue;                             // warp-uniform
            if (r != cur) {
              if (cur >= 0) {
                if constexpr (FX) fx_flush(fx, obase, cur, C, c, lane == 0 && c0 == 0, a0, a1);
                else flush_segment(gbase, obase, cur, C, c, true, lane == 0 && c0 == 0, a0, a1);
              }
              cur = r; a0 = 0.f; a1 = 0.f;
            }
            float f0, f1;
            if (p.feat_nhwc) {
              const float2 v = *reinterpret_cast<const float2*>(s_feat + (h * TW + wl) * kCChunk + 2 * lane);
              f0 = v.x; f1 = v.y;
            } else {
              f0 = s_feat[(2 * lane) * fstride + h * TW + wl];
              f1 = s_feat[(2 * lane + 1) * fstride + h * TW + wl];
            }
            const float q = pr[h];
            a0 = fmaf(q, f0, a0);
            a1 = fmaf(q, f1, a1);
          }
          if (cur >= 0) {
            if constexpr (FX) fx_flush(fx, obase, cur, C, c, lane == 0 && c0 == 0, a0, a1);
            else flush_segment(gbase, obase, cur, C, c, true, lane == 0 && c0 == 0, a0, a1);
          }
        }
      }
    }
    if (c0 + kCChunk < C) {              // next 64 channels: the tile buffer is free once every warp is done with it
      __syncthreads();
      issue_features(c0 + kCChunk);
    }
  }
}

// out[b,t] = out[b,t-1]*discount + grid[b,t]  (stp3.py:296, separate fp32 mul and add like the reference's
// `bev_feature * discount + tmp`).  One CTA = 32 consecutive pillars of one sample; lane = pillar, warp = a group
// of 8 channels, so every global store of the (C, X*Y) output is a fully coalesced 128-byte row segment and no
// shared memory or barrier is needed.  Only occupied (frame, pillar) rows of the scatter grid are read; they are
// zeroed again and their occupancy byte cleared, which leaves the workspace clean for the next call.
// pool_sum (B,S,C) += sum over cells (optional).
// Fixed-point finalize (stp3_lift_splat_fwd_det): what the FX kernels read instead of the fp32 grid.
struct FxGrid {
  long long* grid;          // int64 scatter grid, same layout as the fp32 one
  const unsigned* fmax;     // per-frame bits of m_f
  const unsigned* poison;   // per-frame pillar bitmaps
  int lp;
};

// one int64 grid value of frame scale 2^-k as fp32 (the conversion the deterministic mode defines)
__device__ __forceinline__ float fx_value(long long q, double inv_scale) {
  return __double2float_rn((double)q * inv_scale);
}

__device__ __forceinline__ bool fx_poisoned(const FxGrid& fx, size_t frame, int nvox, int pcell) {
  const size_t words = ((size_t)nvox + 31) / 32;
  return (fx.poison[frame * words + (pcell >> 5)] >> (pcell & 31)) & 1u;
}

template <bool VEC, int SMAX, bool FX>
__global__ void __launch_bounds__(256)
bev_finalize_kernel(float* __restrict__ grid, unsigned char* __restrict__ occ, float* __restrict__ out,
                    float* __restrict__ pool_sum, int S, int C, int nvox, float discount, int out_nhwc,
                    const FxGrid fx) {
  const int b = blockIdx.y;
  const int lane = threadIdx.x;
  const int pcell = blockIdx.x * 32 + lane;
  const int c0 = (blockIdx.z * 8 + threadIdx.y) * 8;
  const bool valid = pcell < nvox && c0 < C;
  // every warp reads the occupancy of its 32 pillars for all frames first (independent loads)
  unsigned occ_bits = 0;
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
    if (t < S && valid && occ[((size_t)b * S + t) * nvox + pcell]) occ_bits |= 1u << t;
  // all grid loads are issued before anything is stored: a store to a line with a load miss in flight would
  // stall the memory pipe (measured: 10x slower), so the re-zeroing happens at the very end
  float v[SMAX][8];
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[t][i] = 0.f;
    if constexpr (FX) {
      if (occ_bits & (1u << t)) {
        const size_t frame = (size_t)b * S + t;
        const long long* src = fx.grid + (frame * nvox + pcell) * C + c0;
        const double inv = pow2d(-slot_exponent(fx.fmax, frame, fx.lp));
        const bool nan = fx_poisoned(fx, frame, nvox, pcell);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (VEC || c0 + i < C) v[t][i] = nan ? __int_as_float(0x7fffffff) : fx_value(__ldcs(src + i), inv);
      }
    } else if (occ_bits & (1u << t)) {
      const float* src = grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
      if (VEC) {
        const float4 lo = __ldcs(reinterpret_cast<const float4*>(src));
        const float4 hi = __ldcs(reinterpret_cast<const float4*>(src + 4));
        v[t][0] = lo.x; v[t][1] = lo.y; v[t][2] = lo.z; v[t][3] = lo.w;
        v[t][4] = hi.x; v[t][5] = hi.y; v[t][6] = hi.z; v[t][7] = hi.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) if (c0 + i < C) v[t][i] = src[i];
      }
    }
  }
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    if (t < S) {
      const size_t bt = (size_t)b * S + t;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(__fmul_rn(acc[i], discount), v[t][i]);
      if (valid) {
        if (out_nhwc == 2) {               // bf16 hi/lo planes for the tensor-core path (VEC only)
          __nv_bfloat16* hp = reinterpret_cast<__nv_bfloat16*>(out) + (bt * nvox + pcell) * C + c0;
          __nv_bfloat16* lp = hp + (size_t)gridDim.y * S * nvox * C;
          uint32_t hw[4], lw[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const __nv_bfloat16 h0 = __float2bfloat16_rn(acc[2 * e]), h1 = __float2bfloat16_rn(acc[2 * e + 1]);
            const __nv_bfloat16 l0 = __float2bfloat16_rn(acc[2 * e] - __bfloat162float(h0));
            const __nv_bfloat16 l1 = __float2bfloat16_rn(acc[2 * e + 1] - __bfloat162float(h1));
            hw[e] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
            lw[e] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
          }
          *reinterpret_cast<uint4*>(hp) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
          *reinterpret_cast<uint4*>(lp) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        } else if (out_nhwc) {
          float* dst = out + (bt * nvox + pcell) * C + c0;
          if (VEC) {
            __stcs(reinterpret_cast<float4*>(dst), make_float4(acc[0], acc[1], acc[2], acc[3]));
            __stcs(reinterpret_cast<float4*>(dst + 4), make_float4(acc[4], acc[5], acc[6], acc[7]));
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) if (c0 + i < C) dst[i] = acc[i];
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (VEC || c0 + i < C) __stcs(out + (bt * C + c0 + i) * (size_t)nvox + pcell, acc[i]);
        }
      }
      if (pool_sum) {    // per-(b,t,c) spatial sum for the pyramid-pooling branch: one partial per CTA, no atomics
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float s = acc[i];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (lane == 0 && c0 + i < C) pool_sum[(((size_t)b * gridDim.x + blockIdx.x) * S + t) * C + c0 + i] = s;
        }
      }
    }
  }
  // leave the workspace clean: re-zero exactly the rows that were read, then the occupancy bytes (after every
  // warp of the CTA has read them)
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    if constexpr (FX) {
      if (occ_bits & (1u << t)) {
        long long* src = fx.grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
#pragma unroll
        for (int i = 0; i < 8; ++i) if (VEC || c0 + i < C) src[i] = 0;
      }
    } else if (occ_bits & (1u << t)) {
      float* src = grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
      if (VEC) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(src) = z;
        *reinterpret_cast<float4*>(src + 4) = z;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) if (c0 + i < C) src[i] = 0.f;
      }
    }
  }
  __syncthreads();
  if (threadIdx.y == 0 && blockIdx.z == gridDim.z - 1) {
    // the last channel-group CTA of these pillars clears the bytes; other groups may still be reading them, so
    // groups > 0 exist only when C > 64 and then the bytes are cleared by a tiny follow-up kernel instead
    for (int t = 0; t < S; ++t)
      if (gridDim.z == 1 && (occ_bits & (1u << t))) occ[((size_t)b * S + t) * nvox + pcell] = 0;
  }
}

// Channels-last outputs (fp32 NHWC, or the bf16 hi/lo planes the tensor-core layers read): one thread = one pillar x
// 16 channels, LPP = C/16 neighbouring lanes cover a pillar.  Every lane moves a full 32-byte sector per access
// (two 128-bit instructions) and the lanes of a pillar touch one contiguous row -- the lane-per-pillar mapping of the kernel
// above would write half sectors 128 bytes apart here.  Same arithmetic, same workspace-cleaning contract; the CTA
// clears the occupancy bytes itself because it covers all channels of its pillars.
// PeerOut (frame-sharded mode, fused with the all-gather): instead of one local tensor the fp32 channels-last rows of
// frame bt go to EVERY rank's gathered (n_frames, nvox, C) buffer, slot first_slot + bt -- plain st.global on
// peer-mapped addresses (NVLink 5 / NVSwitch), so the collective is the kernel's own epilogue and no separate
// all-gather launch follows.
constexpr int kMaxPeers = 8;
struct PeerOut {
  float* ptr[kMaxPeers];
  int n;             // 0: not used (write `out`)
  int first_slot;
};

template <int LPP, int SMAX, bool PEERS, bool FX>
__global__ void __launch_bounds__(256)
bev_finalize_cl_kernel(float* __restrict__ grid, unsigned char* __restrict__ occ, float* __restrict__ out,
                       float* __restrict__ pool_sum, int S, int nvox, float discount, int out_layout,
                       const __grid_constant__ PeerOut peers, const FxGrid fx) {
  constexpr int C = LPP * 16, PPB = 256 / LPP;
  __shared__ float s_pool[8][SMAX][C];
  const int b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = tid % LPP, pcell = blockIdx.x * PPB + tid / LPP;
  const int c0 = sub * 16;
  const bool valid = pcell < nvox;
  unsigned occ_bits = 0;
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
    if (t < S && valid && occ[((size_t)b * S + t) * nvox + pcell]) occ_bits |= 1u << t;
  // every grid load is issued before any store (see above)
  uint32_t v[SMAX][16];
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[t][i] = 0u;
    if constexpr (FX) {
      if (occ_bits & (1u << t)) {
        const size_t frame = (size_t)b * S + t;
        const longlong2* src = reinterpret_cast<const longlong2*>(fx.grid + (frame * nvox + pcell) * C + c0);
        const double inv = pow2d(-slot_exponent(fx.fmax, frame, fx.lp));
        const bool nan = fx_poisoned(fx, frame, nvox, pcell);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const longlong2 q = __ldcs(src + i);
          v[t][2 * i] = nan ? 0x7fffffffu : __float_as_uint(fx_value(q.x, inv));
          v[t][2 * i + 1] = nan ? 0x7fffffffu : __float_as_uint(fx_value(q.y, inv));
        }
      }
    } else if (occ_bits & (1u << t)) {
      const float* src = grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
      uint32_t a[8], c[8];
      ptx::ld_global_v8(src, a);
      ptx::ld_global_v8(src + 8, c);
#pragma unroll
      for (int i = 0; i < 8; ++i) { v[t][i] = a[i]; v[t][8 + i] = c[i]; }
    }
  }
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    if (t < S) {
      const size_t bt = (size_t)b * S + t;
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = __fadd_rn(__fmul_rn(acc[i], discount), __uint_as_float(v[t][i]));
      if (valid) {
        if (out_layout == 2) {
          __nv_bfloat16* hp = reinterpret_cast<__nv_bfloat16*>(out) + (bt * nvox + pcell) * C + c0;
          __nv_bfloat16* lp = hp + (size_t)gridDim.y * S * nvox * C;
          uint32_t hw[8], lw[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float x0 = acc[2 * e], x1 = acc[2 * e + 1];
            const uint32_t h = ptx::pack_bf16x2(x0, x1);
            hw[e] = h;
            lw[e] = ptx::pack_bf16x2(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xFFFF0000u));
          }
          ptx::st_global_v8(hp, hw);
          ptx::st_global_v8(lp, lw);
        } else {
          uint32_t w0[8], w1[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) { w0[i] = __float_as_uint(acc[i]); w1[i] = __float_as_uint(acc[8 + i]); }
          if constexpr (!PEERS) {
            float* dst = out + (bt * nvox + pcell) * C + c0;
            ptx::st_global_v8(dst, w0);
            ptx::st_global_v8(dst + 8, w1);
          } else {
            const size_t off = ((size_t)(peers.first_slot + bt) * nvox + pcell) * C + c0;
#pragma unroll
            for (int q = 0; q < kMaxPeers; ++q) {          // the all-gather: one row to every rank's buffer
              if (q < peers.n) {
                ptx::st_global_v8(peers.ptr[q] + off, w0);
                ptx::st_global_v8(peers.ptr[q] + off + 8, w1);
              }
            }
          }
        }
      }
      if (pool_sum) {
        // sum over the 32/LPP pillars of the warp: halving butterfly (lanes that differ in `off` split the channels)
        float sv[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) sv[i] = acc[i];
        int base = 0;
        int n = 16;
#pragma unroll
        for (int off = LPP; off < 32; off <<= 1) {
          const bool upper = (lane & off) != 0;
          const int half = n >> 1;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (i < half) {
              const float send = upper ? sv[i] : sv[i + half];
              const float keep = upper ? sv[i + half] : sv[i];
              sv[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
          }
          if (upper) base += half;
          n = half;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < n) s_pool[warp][t][c0 + base + i] = sv[i];
      }
    }
  }
  // leave the workspace clean: zero exactly the rows that were read, then the occupancy bytes
  const uint32_t z[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    if (occ_bits & (1u << t)) {
      if constexpr (FX) {
        long long* src = fx.grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
#pragma unroll
        for (int i = 0; i < 4; ++i) ptx::st_global_v8(src + 4 * i, z);
      } else {
        float* src = grid + (((size_t)b * S + t) * nvox + pcell) * C + c0;
        ptx::st_global_v8(src, z);
        ptx::st_global_v8(src + 8, z);
      }
    }
  }
  __syncthreads();
  if (sub == 0)
    for (int t = 0; t < S; ++t)
      if (occ_bits & (1u << t)) occ[((size_t)b * S + t) * nvox + pcell] = 0;
  if (pool_sum) {
    for (int i = tid; i < S * C; i += 256) {
      const int t = i / C, c = i % C;
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) a += s_pool[w][t][c];
      pool_sum[(((size_t)b * gridDim.x + blockIdx.x) * S + t) * C + c] = a;
    }
  }
}

// pool_sum[b,t,c] += sum over a slice of the finalize CTAs' partials (B, nblk, S, C); grid (B*S, kPoolSlices),
// block (32, 8).  All loads of a thread are issued before the partials are zeroed again (the whole workspace stays
// all-zero between calls); pool_sum is cleared by the caller (cudaMemsetAsync in stp3_lift_splat_fwd).
// ORDERED (deterministic mode): each slice stores its sum to slices (B*S, kPoolSlices, C) instead of adding it to out;
// pool_slices_kernel then adds the slices in order.
constexpr int kPoolSlices = 16;
template <bool ORDERED>
__global__ void pool_reduce_kernel(float* __restrict__ part, int nblk, int S, int C, float* __restrict__ out) {
  __shared__ float sm[8][33];
  const int b = blockIdx.x / S, t = blockIdx.x % S;
  const int per = (nblk + kPoolSlices - 1) / kPoolSlices;
  const int k0 = blockIdx.y * per, k1 = min(nblk, k0 + per);
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + threadIdx.x;
    float a = 0.f;
    if (c < C) {
      constexpr int kMaxLoads = 16;
      for (int kb = k0 + threadIdx.y; kb < k1; kb += 8 * kMaxLoads) {
        float v[kMaxLoads];
#pragma unroll
        for (int i = 0; i < kMaxLoads; ++i) {
          const int k = kb + 8 * i;
          v[i] = k < k1 ? part[(((size_t)b * nblk + k) * S + t) * C + c] : 0.f;
        }
#pragma unroll
        for (int i = 0; i < kMaxLoads; ++i) {
          const int k = kb + 8 * i;
          a += v[i];
          if (k < k1) part[(((size_t)b * nblk + k) * S + t) * C + c] = 0.f;
        }
      }
    }
    sm[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
      float tot = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) tot += sm[r][threadIdx.x];
      if constexpr (ORDERED) out[((size_t)blockIdx.x * kPoolSlices + blockIdx.y) * C + c] = tot;
      else atomicAdd(out + (size_t)blockIdx.x * C + c, tot);
    }
    __syncthreads();
  }
}

// pool_sum[f, c] = sum of the kPoolSlices slices of frame f in slice order; re-zeroes the slices
__global__ void pool_slices_kernel(float* __restrict__ slices, int n, int C, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;     // (frame, channel)
  if (i >= n) return;
  const int f = i / C, c = i % C;
  float* s = slices + (size_t)f * kPoolSlices * C + c;
  float v[kPoolSlices];
#pragma unroll
  for (int k = 0; k < kPoolSlices; ++k) v[k] = s[(size_t)k * C];
  float a = 0.f;
#pragma unroll
  for (int k = 0; k < kPoolSlices; ++k) { a += v[k]; s[(size_t)k * C] = 0.f; }
  out[i] = a;
}

// fmax[slot] = bits of the largest finite |x| over the frame's n_per_frame features, for slots blockIdx.y,
// blockIdx.y + gridDim.y, ... < n_frames; the maximum of non-negative float bit patterns is order-independent, so the
// atomicMax is deterministic
__global__ void __launch_bounds__(256)
frame_absmax_kernel(const float* __restrict__ feat, size_t n_per_frame, int n_frames, int vec4,
                    unsigned* __restrict__ fmax) {
  for (int slot = blockIdx.y; slot < n_frames; slot += gridDim.y) {
    const float* x = feat + (size_t)slot * n_per_frame;
    unsigned m = 0;
    auto take = [&](float v) {
      const unsigned b = __float_as_uint(v) & 0x7fffffffu;
      if (b < 0x7f800000u) m = max(m, b);
    };
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    if (vec4) {
      const float4* x4 = reinterpret_cast<const float4*>(x);
      for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per_frame / 4; i += stride) {
        const float4 v = __ldg(x4 + i);
        take(v.x); take(v.y); take(v.z); take(v.w);
      }
    } else {
      for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per_frame; i += stride) take(__ldg(x + i));
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(fmax + slot, m);
  }
}

// C > 64 only: occupancy bytes are cleared after every channel group has consumed them
__global__ void clear_bytes_kernel(unsigned char* __restrict__ p, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i * 16 < n) reinterpret_cast<uint4*>(p)[i] = make_uint4(0, 0, 0, 0);
}

}  // namespace stp3

using namespace stp3;

static size_t grid_bytes(int B, int S, int C, int nx, int ny) {
  const size_t g = (size_t)B * S * nx * ny * C * sizeof(float);
  return (g + 255) & ~(size_t)255;
}

static size_t occ_bytes(int B, int S, int nx, int ny) { return ((size_t)B * S * nx * ny + 255) & ~(size_t)255; }

static size_t workspace_bytes_for(int B, int S, int C, int nx, int ny) {
  if (B <= 0 || S <= 0 || C <= 0 || nx <= 0 || ny <= 0) return 0;
  const size_t part = (((size_t)B * ceil_div(nx * ny, 32) * S * C * sizeof(float)) + 255) & ~(size_t)255;
  return grid_bytes(B, S, C, nx, ny) + occ_bytes(B, S, nx, ny) + part;   // scatter grid | occupancy | pool partials
}

// frame mode lays its f_count raw frames out as f_count samples of one frame
extern "C" size_t stp3_lift_splat_workspace_bytes(const stp3_lift_splat_desc* desc) {
  if (!desc || desc->f_count < 0) return 0;
  const bool raw = desc->f_count > 0;
  return workspace_bytes_for(raw ? desc->f_count : desc->B, raw ? 1 : desc->S, desc->C, desc->nx, desc->ny);
}

// Workspace of stp3_lift_splat_fwd_det, byte offsets:
//   int64 scatter grid | occupancy | pool partials | m_f bits (per frame) | poison bitmaps | pool slices
// The grid alone is twice the fp32 one, so the total is above stp3_lift_splat_workspace_bytes and one zeroed buffer
// serves both modes.
namespace {
struct DetLayout {
  size_t occ, part, fmax, poison, slices, total;
};

DetLayout det_layout(int B, int S, int C, int nx, int ny) {
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t frames = (size_t)B * S, nvox = (size_t)nx * ny;
  DetLayout L;
  size_t o = al(frames * nvox * C * sizeof(long long));
  L.occ = o;    o += occ_bytes(B, S, nx, ny);
  L.part = o;   o += al((size_t)B * ceil_div(nx * ny, 32) * S * C * sizeof(float));
  L.fmax = o;   o += al(frames * sizeof(unsigned));
  L.poison = o; o += al(frames * ((nvox + 31) / 32) * sizeof(unsigned));
  L.slices = o; o += al(frames * kPoolSlices * C * sizeof(float));
  L.total = o;
  return L;
}

DetLayout det_layout(const stp3_lift_splat_desc* d) {
  const bool raw = d->f_count > 0;
  return det_layout(raw ? d->f_count : d->B, raw ? 1 : d->S, d->C, d->nx, d->ny);
}
}  // namespace

extern "C" size_t stp3_lift_splat_det_workspace_bytes(const stp3_lift_splat_desc* desc) {
  if (!desc || desc->f_count < 0 || desc->B <= 0 || desc->S <= 0 || desc->C <= 0 || desc->nx <= 0 || desc->ny <= 0)
    return 0;
  return det_layout(desc).total;
}

extern "C" int stp3_lift_splat_workspace_init(void* workspace, size_t workspace_bytes, void* stream) {
  STP3_CHECK_ARG(workspace != nullptr, "stp3_lift_splat_workspace_init: null workspace");
  STP3_CUDA_OK(cudaMemsetAsync(workspace, 0, workspace_bytes, reinterpret_cast<cudaStream_t>(stream)));
  return STP3_OK;
}

int stp3::check_lift_splat_desc(const char* fn, const stp3_lift_splat_desc* d, const float* feat,
                                const float* depth_logits, int max_frames, BevQuant& q) {
  STP3_CHECK_ARG(d && feat && d->cam_M && d->cam_t && d->ego_R && d->ego_t && d->xs && d->ys && d->ds,
                 "%s: null pointer argument", fn);
  STP3_CHECK_ARG(d->use_depth_distribution == 0 || depth_logits, "depth_logits is NULL but use_depth_distribution=1");
  STP3_CHECK_ARG(d->B > 0 && d->S > 0 && d->N > 0 && d->D > 0 && d->Hf > 0 && d->Wf > 0 && d->C > 0, "non-positive dimension");
  STP3_CHECK_ARG(d->S <= max_frames, "receptive field S=%d exceeds the supported %d", d->S, max_frames);
  STP3_CHECK_ARG(d->nx > 0 && d->ny > 0, "empty BEV grid");
  STP3_CHECK_ARG(d->nz == 1, "nz=%d: the reference (stp3.py:298) and this kernel support a single height bin", d->nz);
  STP3_CHECK_ARG((long long)d->nx * d->ny * d->nz < (1ll << 31), "BEV grid too large for int32 ranks");
  STP3_CHECK_ARG(d->feat_layout == 0 || d->feat_layout == 1, "feat_layout must be 0 (NCHW) or 1 (NHWC)");
  STP3_CHECK_ARG(d->f_count == 0 ? d->f_begin == 0
                                 : d->f_begin >= 0 && d->f_count > 0 && (long long)d->f_begin + d->f_count <= (long long)d->B * d->S,
                 "frame range outside [0, B*S)");
  for (int i = 0; i < 3; ++i) {
    q.off[i] = d->bev_off[i]; q.res[i] = d->bev_res[i];
    int e = 0;
    const float m = frexpf(d->bev_res[i], &e);       // res = m * 2^e ; power of two <=> m == 0.5
    q.inv_ok[i] = (m == 0.5f && e > -100 && e < 100) ? 1 : 0;
    q.inv[i] = q.inv_ok[i] ? ldexpf(1.0f, 1 - e) : 0.f;
  }
  q.nx = d->nx; q.ny = d->ny; q.nz = d->nz;
  return STP3_OK;
}

// The scatter and finalize launches of one forward call: the public plan plus what the launch needs beyond it.
namespace {
struct LiftLaunch {
  stp3_lift_splat_kernel_plan plan;
  LiftSplatTmaMaps maps;   // valid when plan.scatter == 1
  size_t smem;             // generic scatter kernel
  size_t smem_tma;         // TMA scatter kernel
};

// The one place that decides which kernels run (stp3_lift_splat_plan, stp3_lift_splat_fwd).  Checks the descriptor and
// the output choice; host only -- the tensor-map encode reads nothing behind the pointers.
int plan_lift_splat(const char* fn, const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                    int out_layout, int n_peers, BevQuant& q, LiftLaunch& L) {
  if (const int rc = check_lift_splat_desc(fn, desc, feat, depth_logits, kMaxFrames, q)) return rc;
  const int B = desc->B, S = desc->S, N = desc->N, D = desc->D, Hf = desc->Hf, Wf = desc->Wf, C = desc->C;
  const int feat_layout = desc->feat_layout;
  const bool raw = desc->f_count > 0;
  const int Sw = raw ? 1 : S;                                   // frames per sample of the scatter grid / finalize
  STP3_CHECK_ARG(n_peers >= 0 && n_peers <= kMaxPeers, "n_peers must be in [0, %d], with peer_out when it is not 0",
                 kMaxPeers);
  STP3_CHECK_ARG(raw || n_peers == 0, "peer outputs need frame mode (f_count > 0)");
  STP3_CHECK_ARG(out_layout >= 0 && out_layout <= 2, "out_layout must be 0 (C,X,Y), 1 (X,Y,C) or 2 (bf16 hi/lo X,Y,C)");
  STP3_CHECK_ARG(!raw || out_layout == 1, "frame mode writes fp32 channels-last frames (out_layout 1)");
  STP3_CHECK_ARG(n_peers == 0 || C == 32 || C == 64 || C == 128,
                 "peer outputs need C in {32, 64, 128} (channels-last finalize kernel)");
  STP3_CHECK_ARG(out_layout != 2 || C % 8 == 0, "out_layout 2 needs C %% 8 == 0");
  stp3_lift_splat_kernel_plan& P = L.plan;
  memset(&P, 0, sizeof(P));

  // generic scatter: tile width as wide as shared memory allows (<= 4 columns), at least 1
  const int HP = (Hf + 3) & ~3;
  auto smem_for = [&](int tw) {
    return (size_t)D * tw * HP * 8 + (size_t)D * tw * 4 +
           (size_t)(kCChunk * ((((Hf + kHChunk - 1) / kHChunk) * kHChunk * tw) | 1) + 12 * kMaxFrames + Hf + D +
                    kScatterThreads) * sizeof(float);
  };
  int TW = 4;
  while (TW > 1 && smem_for(TW) > 110 * 1024) TW >>= 1;
  L.smem = smem_for(TW);
  STP3_CHECK_ARG(L.smem <= 227 * 1024, "D*Hf = %d too large for one image column in shared memory", D * Hf);
  P.scatter_tw = TW;

  // TMA-staged scatter: 16-byte aligned rows for the tensor maps, whole 64-channel chunks for the fixed transaction
  // counts, two mma k-steps (Hf <= 32), and a tile that leaves room for two CTAs per SM
  const int npix = Hf * kTmaTW, feat_floats = npix * kCChunk;
  L.smem_tma = 128 + ((size_t)((D * npix + 31) & ~31) + ((feat_floats + 31) & ~31) + 2 * (size_t)D * kTmaTW * HP +
                      (kSegPasses + 1) * (size_t)D * kTmaTW + 4 + 12 * kMaxFrames + Hf + D + kScatterThreads + 2) * 4 + 16;
  static const int no_tma = [] { const char* e = getenv("STP3_LIFT_NO_TMA"); return e ? atoi(e) : 0; }();
  P.tma_rules = !no_tma && TW == kTmaTW && Wf % 4 == 0 && C % kCChunk == 0 && D <= 256 && Hf <= 32 &&
                (reinterpret_cast<uintptr_t>(feat) & 15) == 0 &&
                (!depth_logits || (reinterpret_cast<uintptr_t>(depth_logits) & 15) == 0) && L.smem_tma <= 113 * 1024;
  if (P.tma_rules) {
    const TmapEncodeFn enc = tmap_encode_fn();
    if (enc) {   // otherwise (or when an encode fails) the generic kernel runs
      const long long n_img = (long long)B * S * N;
      const cuuint32_t es[3] = {1, 1, 1};
      CUresult r1 = CUDA_SUCCESS, r2;
      if (desc->use_depth_distribution) {
        const cuuint64_t dims[3] = {(cuuint64_t)Wf, (cuuint64_t)Hf, (cuuint64_t)(D * n_img)};
        const cuuint64_t strides[2] = {(cuuint64_t)Wf * 4, (cuuint64_t)Hf * Wf * 4};
        const cuuint32_t box[3] = {4, (cuuint32_t)Hf, (cuuint32_t)D};
        r1 = enc(&L.maps.depth, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(depth_logits), dims, strides, box,
                 es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      } else {
        memset(&L.maps.depth, 0, sizeof(L.maps.depth));
      }
      if (feat_layout == 0) {
        const cuuint64_t dims[3] = {(cuuint64_t)Wf, (cuuint64_t)Hf, (cuuint64_t)(C * n_img)};
        const cuuint64_t strides[2] = {(cuuint64_t)Wf * 4, (cuuint64_t)Hf * Wf * 4};
        const cuuint32_t box[3] = {4, (cuuint32_t)Hf, (cuuint32_t)kCChunk};
        r2 = enc(&L.maps.feat, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(feat), dims, strides, box, es,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      } else {
        const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)Wf, (cuuint64_t)(Hf * n_img)};
        const cuuint64_t strides[2] = {(cuuint64_t)C * 4, (cuuint64_t)Wf * C * 4};
        const cuuint32_t box[3] = {(cuuint32_t)kCChunk, 4, (cuuint32_t)Hf};
        r2 = enc(&L.maps.feat, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(feat), dims, strides, box, es,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      }
      P.scatter = r1 == CUDA_SUCCESS && r2 == CUDA_SUCCESS;
    }
  }

  // finalize: channels-last outputs with 32 / 64 / 128 channels and few frames take the sector-exact kernel
  // (one thread = 16 channels); everything else the lane-per-pillar kernel (8 warps x 8 channels per CTA)
  P.finalize = out_layout != 0 && (C == 32 || C == 64 || C == 128) && Sw <= 4;
  if (P.finalize) {
    P.finalize_smax = 4;
    P.finalize_lpp = C / 16;
    P.channel_groups = 1;
  } else {
    P.finalize_vec = C % 8 == 0;
    P.finalize_smax = Sw <= 4 ? 4 : 8;
    P.channel_groups = ceil_div(C, 64);
  }
  return STP3_OK;
}
}  // namespace

extern "C" int stp3_lift_splat_plan(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                                    int out_layout, int n_peers, stp3_lift_splat_kernel_plan* plan) {
  STP3_CHECK_ARG(plan != nullptr, "stp3_lift_splat_plan: null plan");
  BevQuant q;
  LiftLaunch L;
  if (const int rc = plan_lift_splat("stp3_lift_splat_plan", desc, feat, depth_logits, out_layout, n_peers, q, L))
    return rc;
  *plan = L.plan;
  return STP3_OK;
}

// f_count == 0: all B*S frames, discount recurrence over each sample's S frames.  f_count > 0: frame-sharded call --
// only the flat frames f_begin + [0, f_count) are splatted and written RAW (no recurrence), one (nx, ny, C) grid per
// frame, to `out` or to every peer's gathered buffer; the caller all-gathers them and applies stp3_bev_discount.
// det: the fixed-point form (stp3_lift_splat_fwd_det) -- the same plan's kernels with FX set, after the m_f pre-pass,
// and the pool slices added in order.
static int lift_splat_fwd(bool det, const char* fn, const stp3_lift_splat_desc* desc, const float* feat,
                          const float* depth_logits, int32_t* ranks_out, float* pool_sum, void* workspace,
                          size_t workspace_bytes, float* out, int out_layout, int n_peers, void* const* peer_out,
                          void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  BevQuant q;
  LiftLaunch L;
  if (const int rc = plan_lift_splat(fn, desc, feat, depth_logits, out_layout, n_peers, q, L))
    return rc;
  const stp3_lift_splat_kernel_plan& P = L.plan;
  const int nx = desc->nx, ny = desc->ny, nz = desc->nz;
  const int B = desc->B, S = desc->S, N = desc->N, D = desc->D, Hf = desc->Hf, Wf = desc->Wf, C = desc->C;
  const bool raw = desc->f_count > 0;
  const float discount = raw ? 0.f : desc->discount;
  const int Bw = raw ? desc->f_count : B, Sw = raw ? 1 : S;     // shape of the scatter grid / finalize launch
  STP3_CHECK_ARG(n_peers == 0 || peer_out, "n_peers must be in [0, %d], with peer_out when it is not 0", kMaxPeers);
  STP3_CHECK_ARG((out || n_peers > 0) && workspace, "%s: null pointer argument", fn);
  STP3_CHECK_ARG(!raw || (!ranks_out && !pool_sum), "frame mode writes no ranks_out or pool_sum");
  PeerOut po;
  po.n = n_peers; po.first_slot = desc->f_begin;
  for (int i = 0; i < kMaxPeers; ++i) po.ptr[i] = i < n_peers ? static_cast<float*>(peer_out[i]) : nullptr;
  for (int i = 0; i < n_peers; ++i)
    STP3_CHECK_ARG(po.ptr[i] && (reinterpret_cast<uintptr_t>(po.ptr[i]) & 31) == 0, "peer buffer %d is null or not 32-byte aligned", i);
  STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  const size_t need = det ? stp3_lift_splat_det_workspace_bytes(desc) : stp3_lift_splat_workspace_bytes(desc);
  if (workspace_bytes < need) return set_error(STP3_ENOSPC, "workspace too small: %zu < %zu", workspace_bytes, need);

  LiftSplatParams p;
  p.f_begin = desc->f_begin;
  p.feat = feat; p.depth = depth_logits; p.cam_M = desc->cam_M; p.cam_t = desc->cam_t; p.ego_R = desc->ego_R;
  p.ego_t = desc->ego_t; p.xs = desc->xs; p.ys = desc->ys; p.ds = desc->ds;
  for (int i = 0; i < 3; ++i) { p.off[i] = q.off[i]; p.res[i] = q.res[i]; p.inv[i] = q.inv[i]; p.inv_ok[i] = q.inv_ok[i]; }
  p.nx = nx; p.ny = ny; p.nz = nz;
  p.B = B; p.S = S; p.N = N; p.D = D; p.Hf = Hf; p.Wf = Wf; p.C = C;
  p.feat_nhwc = desc->feat_layout; p.use_depth = desc->use_depth_distribution;
  p.ranks_out = ranks_out;
  p.grid = static_cast<float*>(workspace);
  p.occ = static_cast<unsigned char*>(workspace) + grid_bytes(Bw, Sw, C, nx, ny);
  p.TW = P.scatter_tw;
  p.tiles_w = ceil_div(Wf, P.scatter_tw);
  const long long nblk = (long long)Bw * Sw * N * p.tiles_w;
  STP3_CHECK_ARG(nblk < (1ll << 31), "grid too large");
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const DetLayout DL = det_layout(desc);
  FxGrid fx;
  memset(&fx, 0, sizeof(fx));
  p.qgrid = nullptr; p.fmax = nullptr; p.poison = nullptr; p.lp = 0;
  if (det) {
    const long long points = (long long)N * D * Hf * Wf;
    while ((1ll << p.lp) < points) ++p.lp;
    p.grid = nullptr;
    p.qgrid = reinterpret_cast<long long*>(ws);
    p.occ = ws + DL.occ;
    p.fmax = reinterpret_cast<unsigned*>(ws + DL.fmax);
    p.poison = reinterpret_cast<unsigned*>(ws + DL.poison);
    fx.grid = p.qgrid; fx.fmax = p.fmax; fx.poison = p.poison; fx.lp = p.lp;
    // m_f of every frame of the launch (its features are one contiguous block in both layouts)
    const size_t per_frame = (size_t)N * C * Hf * Wf;
    const int vec4 = per_frame % 4 == 0 && (reinterpret_cast<uintptr_t>(feat) & 15) == 0;
    const size_t work = vec4 ? per_frame / 4 : per_frame;
    const unsigned gx = (unsigned)std::max<size_t>(1, std::min<size_t>(1024, (work + 2047) / 2048));
    const int frames = Bw * Sw;     // grid.y is capped at 65535; the kernel loops over the frames beyond
    frame_absmax_kernel<<<dim3(gx, std::min(frames, 65535)), 256, 0, stream>>>(
        feat + (size_t)desc->f_begin * per_frame, per_frame, frames, vec4, reinterpret_cast<unsigned*>(ws + DL.fmax));
    STP3_CUDA_OK(cudaGetLastError());
  }

  if (P.scatter) {
    auto tma = det ? lift_splat_scatter_tma_kernel<true> : lift_splat_scatter_tma_kernel<false>;
    STP3_CUDA_OK(cudaFuncSetAttribute(tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem_tma));
    tma<<<(unsigned)nblk, kScatterThreads, L.smem_tma, stream>>>(L.maps, p);
  } else {
    auto launch = [&](auto kernel) -> int {
      STP3_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
      kernel<<<(unsigned)nblk, kScatterThreads, L.smem, stream>>>(p);
      return STP3_OK;
    };
    int rc;
    if (det)
      rc = P.scatter_tw == 4 ? launch(lift_splat_scatter_kernel<4, true>)
         : P.scatter_tw == 2 ? launch(lift_splat_scatter_kernel<2, true>) : launch(lift_splat_scatter_kernel<1, true>);
    else
      rc = P.scatter_tw == 4 ? launch(lift_splat_scatter_kernel<4, false>)
         : P.scatter_tw == 2 ? launch(lift_splat_scatter_kernel<2, false>) : launch(lift_splat_scatter_kernel<1, false>);
    if (rc != STP3_OK) return rc;
  }
  STP3_CUDA_OK(cudaGetLastError());

  const int nvox = nx * ny * nz;
  float* pool_part = pool_sum ? reinterpret_cast<float*>(det ? ws + DL.part : p.occ + occ_bytes(Bw, Sw, nx, ny)) : nullptr;
  int pool_blocks = ceil_div(nvox, 32);
  if (P.finalize) {
    pool_blocks = ceil_div(nvox, 256 / P.finalize_lpp);
    dim3 cgrid(pool_blocks, Bw);
#define STP3_FIN_CL(LPP_, PEERS_, FX_) \
    bev_finalize_cl_kernel<LPP_, 4, PEERS_, FX_><<<cgrid, 256, 0, stream>>>(p.grid, p.occ, out, pool_part, Sw, nvox, discount, out_layout, po, fx)
#define STP3_FIN_CL_LPP(PEERS_, FX_) \
    do { \
      if (P.finalize_lpp == 2) STP3_FIN_CL(2, PEERS_, FX_); else if (P.finalize_lpp == 4) STP3_FIN_CL(4, PEERS_, FX_); \
      else STP3_FIN_CL(8, PEERS_, FX_); \
    } while (0)
    if (det) { if (po.n > 0) STP3_FIN_CL_LPP(true, true); else STP3_FIN_CL_LPP(false, true); }
    else     { if (po.n > 0) STP3_FIN_CL_LPP(true, false); else STP3_FIN_CL_LPP(false, false); }
#undef STP3_FIN_CL_LPP
#undef STP3_FIN_CL
  } else {
    dim3 fgrid(pool_blocks, Bw, P.channel_groups), fblock(32, C >= 64 ? 8 : ceil_div(C, 8));
#define STP3_FINALIZE(VEC, SMAX, FX_) \
  bev_finalize_kernel<VEC, SMAX, FX_><<<fgrid, fblock, 0, stream>>>(p.grid, p.occ, out, pool_part, Sw, C, nvox, discount, out_layout, fx)
#define STP3_FINALIZE_ANY(FX_) \
    do { \
      if (P.finalize_vec) { if (P.finalize_smax == 4) STP3_FINALIZE(true, 4, FX_); else STP3_FINALIZE(true, 8, FX_); } \
      else                { if (P.finalize_smax == 4) STP3_FINALIZE(false, 4, FX_); else STP3_FINALIZE(false, 8, FX_); } \
    } while (0)
    if (det) STP3_FINALIZE_ANY(true); else STP3_FINALIZE_ANY(false);
#undef STP3_FINALIZE_ANY
#undef STP3_FINALIZE
  }
  STP3_CUDA_OK(cudaGetLastError());
  if (pool_sum && det) {
    float* slices = reinterpret_cast<float*>(ws + DL.slices);
    pool_reduce_kernel<true><<<dim3(Bw * Sw, kPoolSlices), dim3(32, 8), 0, stream>>>(pool_part, pool_blocks, Sw, C, slices);
    STP3_CUDA_OK(cudaGetLastError());
    const int n = Bw * Sw * C;
    pool_slices_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(slices, n, C, pool_sum);
    STP3_CUDA_OK(cudaGetLastError());
  } else if (pool_sum) {
    STP3_CUDA_OK(cudaMemsetAsync(pool_sum, 0, (size_t)Bw * Sw * C * sizeof(float), stream));
    pool_reduce_kernel<false><<<dim3(Bw * Sw, kPoolSlices), dim3(32, 8), 0, stream>>>(pool_part, pool_blocks, Sw, C, pool_sum);
    STP3_CUDA_OK(cudaGetLastError());
  }
  if (P.channel_groups > 1) {
    const size_t nocc = ((size_t)Bw * Sw * nvox + 255) & ~(size_t)255;
    clear_bytes_kernel<<<(unsigned)((nocc / 16 + 255) / 256), 256, 0, stream>>>(p.occ, nocc);
    STP3_CUDA_OK(cudaGetLastError());
  }
  if (det)   // the m_f bits and the poison bitmaps: everything else was re-zeroed by the kernels that read it
    STP3_CUDA_OK(cudaMemsetAsync(ws + DL.fmax, 0, DL.slices - DL.fmax, stream));
  return STP3_OK;
}

extern "C" int stp3_lift_splat_fwd(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                                   int32_t* ranks_out, float* pool_sum, void* workspace, size_t workspace_bytes,
                                   float* out, int out_layout, int n_peers, void* const* peer_out, void* stream) {
  return lift_splat_fwd(false, "stp3_lift_splat_fwd", desc, feat, depth_logits, ranks_out, pool_sum, workspace,
                        workspace_bytes, out, out_layout, n_peers, peer_out, stream);
}

extern "C" int stp3_lift_splat_fwd_det(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                                       int32_t* ranks_out, float* pool_sum, void* workspace, size_t workspace_bytes,
                                       float* out, int out_layout, int n_peers, void* const* peer_out, void* stream) {
  return lift_splat_fwd(true, "stp3_lift_splat_fwd_det", desc, feat, depth_logits, ranks_out, pool_sum, workspace,
                        workspace_bytes, out, out_layout, n_peers, peer_out, stream);
}

namespace stp3 {
// out[b,t] = out[b,t-1]*discount + raw[b,t] over channels-last fp32 raw splats, written as bf16 hi/lo planes
// (the discount recurrence of stp3.py:296 applied after the frames were all-gathered); one thread = 8 channels of a cell
__global__ void __launch_bounds__(256)
bev_discount_kernel(const float* __restrict__ raw, int S, size_t cells8, float discount, __nv_bfloat16* __restrict__ hi,
                    __nv_bfloat16* __restrict__ lo, size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const size_t b = idx / cells8, r = idx % cells8;       // r = (cell, 8-channel group) within one frame
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int t = 0; t < S; ++t) {
    const size_t off = ((b * S + t) * cells8 + r) * 8;
    const float4 a = __ldcs(reinterpret_cast<const float4*>(raw + off));
    const float4 c = __ldcs(reinterpret_cast<const float4*>(raw + off) + 1);
    const float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      acc[2 * e] = __fadd_rn(__fmul_rn(acc[2 * e], discount), v[2 * e]);
      acc[2 * e + 1] = __fadd_rn(__fmul_rn(acc[2 * e + 1], discount), v[2 * e + 1]);
      const uint32_t h = ptx::pack_bf16x2(acc[2 * e], acc[2 * e + 1]);
      hw[e] = h;
      lw[e] = ptx::pack_bf16x2(acc[2 * e] - __uint_as_float(h << 16), acc[2 * e + 1] - __uint_as_float(h & 0xFFFF0000u));
    }
    *reinterpret_cast<uint4*>(hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
}
}  // namespace stp3

extern "C" int stp3_bev_discount(const float* raw, int B, int S, int nx, int ny, int C, float discount, void* out_hi,
                                 void* out_lo, void* stream) {
  STP3_CHECK_ARG(raw && out_hi && out_lo && B > 0 && S > 0 && nx > 0 && ny > 0 && C > 0 && C % 8 == 0,
                 "stp3_bev_discount: bad argument (C must be a multiple of 8)");
  const size_t cells8 = (size_t)nx * ny * (C / 8);
  const size_t total = (size_t)B * cells8;
  bev_discount_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      raw, S, cells8, discount, static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), total);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
