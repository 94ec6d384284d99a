// Train-mode pieces of the dense path (the BEV decoder, stp3/models/decoder.py, and the DeepLab head,
// convolutions.py:272-280): convolution weight gradient (dilated too), BatchNorm with batch statistics (stats / apply with
// fused dropout / backward), per-image channel sums, fp32 bilinear x2 and its backward, the interleave of the four
// stride-2 input-gradient phases, and the sigmoid backward.  Tensors are fp32 channels-last (n_pix, cstride) unless
// noted.  Every reduction is deterministic: per-block partials go to caller scratch and are summed in a fixed order
// (no float atomics), and the block decomposition depends only on the problem shape, so two calls on the same inputs
// return bitwise-identical results.
#include <climits>
#include <type_traits>

#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

// ------------------------------------------------------------------------------------------------ weight gradient
// dW[co][ci][ky][kx] = sum over output pixels p of g[p][co] * x[p * stride + (ky*d - pad, kx*d - pad)][ci]  (zero outside)
// as a GEMM on the tensor cores: M = co, N = ci, K = output pixels.  Both operands are channels-last, i.e. MN-major for
// this GEMM: a K row (one pixel) holds 64 consecutive co (A) or ci (B).  One CTA = one warpgroup = one tap x 64 co x
// 64 ci x one contiguous range of output pixels (the K split).  Each 64-pixel stage is staged as bf16 hi / lo planes
// in the 128-byte swizzled layout (the fp32 -> hi/lo split happens on the way in; the shifted, strided window of x
// reads zeros outside the image) and multiplied by wgmma with the transpose bits set, three products per pair
// (hi*hi + hi*lo + lo*hi, fp32 accumulate in registers) like every product of this library.
constexpr int kWgTile = 64, kWgK = 64;
constexpr int kWgTileBytes = kWgK * kWgTile * 2;          // one bf16 plane of one operand: 64 pixels x 128 B

// n_img = B * T images, frame-major within a sample; kt > 1: causal time taps, output frame t of a sample reads frame
// t + it - (kt - 1) of the same sample (frames outside [0, T) are zeros).  T = kt = 1 is the 2-D convolution.
struct WgradShape {
  int n_img, H, W, x_cstride, cin, Ho, Wo, g_cstride, cout, stride, kh, kw, pad, dil;
  int T = 1, kt = 1;
};

// does an output axis of n_out positions, read at o * stride + d, touch the input extent [0, n_in) at all?
__device__ __forceinline__ bool tap_in_image(int d, int n_out, int stride, int n_in) {
  const int o = d >= 0 ? 0 : (-d + stride - 1) / stride;       // first o with o * stride + d >= 0
  return o < n_out && o * stride + d < n_in;
}

__host__ __device__ inline long long wgrad_pixels(const WgradShape& s) { return (long long)s.n_img * s.Ho * s.Wo; }

// the K split: a function of the shape only (determinism), ~4 CTAs per SM of an H100, >= 256 pixels per CTA
inline int wgrad_splits(const WgradShape& s) {
  const long long tiles = (long long)s.kt * s.kh * s.kw * ceil_div(s.cout, kWgTile) * ceil_div(s.cin, kWgTile);
  const long long px = wgrad_pixels(s);
  long long n = (132 * 4 + tiles - 1) / tiles;
  const long long max_by_px = (px + 255) / 256;
  if (n > max_by_px) n = max_by_px;
  if (n < 1) n = 1;
  if (n > 1024) n = 1024;
  return (int)n;
}

// 8 consecutive fp32 channels [c0, c0 + 8) of row `row` (NULL row = zeros) -> bf16 hi / lo, one 16-byte chunk each
__device__ __forceinline__ void load8_split(const float* row, int c0, int C, bool vec, uint4& hi, uint4& lo) {
  float v[8];
  if (row && vec && c0 + 8 <= C) {
    const float4 a = *reinterpret_cast<const float4*>(row + c0), b = *reinterpret_cast<const float4*>(row + c0 + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (row && c0 + i < C) ? row[c0 + i] : 0.f;
  }
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) ptx::split_hilo(v[2 * e], v[2 * e + 1], h[e], l[e]);
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// 8 consecutive 16-bit channels [c0, c0 + 8) of row `row` (NULL row = zeros), one 16-byte chunk
__device__ __forceinline__ uint4 load8_plane(const uint16_t* row, int c0, int C, bool vec) {
  if (row && vec && c0 + 8 <= C) return *reinterpret_cast<const uint4*>(row + c0);
  uint32_t h[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const uint32_t a = (row && c0 + 2 * e < C) ? row[c0 + 2 * e] : 0u;
    const uint32_t b = (row && c0 + 2 * e + 1 < C) ? row[c0 + 2 * e + 1] : 0u;
    h[e] = a | (b << 16);
  }
  return make_uint4(h[0], h[1], h[2], h[3]);
}

// OP 0: x and g fp32, split into hi / lo on the way in, three products per pair.  OP 1 / 2 (the one-product mode of
// stp3_conv_wgrad_plane): x and g are one bf16 / fp16 plane each, staged as they are, one product per pair.
template <int OP>
__global__ void __launch_bounds__(128, 1)
wgrad_partial_kernel(const std::conditional_t<OP == 0, float, uint16_t>* __restrict__ x,
                     const std::conditional_t<OP == 0, float, uint16_t>* __restrict__ g, WgradShape s,
                     long long px_per_split, int vec_x, int vec_g, float* __restrict__ part) {
  using In = std::conditional_t<OP == 0, float, uint16_t>;
  extern __shared__ uint8_t wg_smem_raw[];
  // four 8 KB planes, 1024-byte aligned (the swizzle atom): A hi, A lo (g), B hi, B lo (x); OP != 0: A (g), B (x)
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~uintptr_t(1023));
  const int co_tiles = (s.cout + kWgTile - 1) / kWgTile, ci_tiles = (s.cin + kWgTile - 1) / kWgTile;
  int t = blockIdx.y;
  const int cit = t % ci_tiles; t /= ci_tiles;
  const int cot = t % co_tiles; t /= co_tiles;
  const int tap = t;                                   // (it * kh + ky) * kw + kx
  const int dy = tap / s.kw % s.kh * s.dil - s.pad, dx = tap % s.kw * s.dil - s.pad;
  const int dt = tap / (s.kw * s.kh) - (s.kt - 1);     // <= 0: causal
  // a tap whose window lies in the zero padding for every output pixel (large dilations on small maps, a time offset
  // of T frames or more) contributes exact zeros: the CTA stores them without streaming the pixels
  const bool live = tap_in_image(dy, s.Ho, s.stride, s.H) && tap_in_image(dx, s.Wo, s.stride, s.W) && -dt < s.T;
  const long long P = wgrad_pixels(s);
  const long long p_begin = (long long)blockIdx.x * px_per_split;
  const long long p_end = p_begin + px_per_split < P ? p_begin + px_per_split : P;
  const int tid = threadIdx.x;
  const int co0 = cot * kWgTile, ci0 = cit * kWgTile;
  const uint32_t s_base = ptx::smem_u32(sm);
  // each 64-pixel stage is multiplied into `stage` (its first wgmma overwrites it) and then added to `acc` with an
  // ordinary fp32 add: the tensor cores' accumulation does not round to nearest, and chained over a whole split (up to
  // thousands of pixels) its error grew with the pixels per split (DESIGN 3.10); chained over one stage it is negligible
  float acc[32], stage[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = stage[i] = 0.f;
  for (long long p0 = p_begin; live && p0 < p_end; p0 += kWgK) {
    // stage: 64 pixel rows x 8 chunks of 8 channels, per operand; chunk c of row r lives at chunk c ^ (r % 8)
#pragma unroll
    for (int k = 0; k < (kWgK * 8) / 128; ++k) {
      const int idx = tid + 128 * k;
      const int r = idx >> 3, c = idx & 7;
      const long long p = p0 + r;
      const In* grow = nullptr;
      const In* xrow = nullptr;
      if (p < p_end) {
        const int ox = (int)(p % s.Wo);
        const long long q = p / s.Wo;
        const int oy = (int)(q % s.Ho);
        const long long img = q / s.Ho;
        grow = g + p * s.g_cstride + co0;
        const int iy = oy * s.stride + dy, ix = ox * s.stride + dx, it = (int)(img % s.T) + dt;
        if (iy >= 0 && iy < s.H && ix >= 0 && ix < s.W && it >= 0)
          xrow = x + (((img + dt) * s.H + iy) * s.W + ix) * s.x_cstride + ci0;
      }
      const int off = r * 128 + ((c ^ (r & 7)) << 4);
      if constexpr (OP == 0) {
        uint4 gh, gl, xh, xl;
        load8_split(grow, c * 8, s.cout - co0, vec_g, gh, gl);
        load8_split(xrow, c * 8, s.cin - ci0, vec_x, xh, xl);
        *reinterpret_cast<uint4*>(sm + 0 * kWgTileBytes + off) = gh;
        *reinterpret_cast<uint4*>(sm + 1 * kWgTileBytes + off) = gl;
        *reinterpret_cast<uint4*>(sm + 2 * kWgTileBytes + off) = xh;
        *reinterpret_cast<uint4*>(sm + 3 * kWgTileBytes + off) = xl;
      } else {
        *reinterpret_cast<uint4*>(sm + 0 * kWgTileBytes + off) = load8_plane(grow, c * 8, s.cout - co0, vec_g);
        *reinterpret_cast<uint4*>(sm + 1 * kWgTileBytes + off) = load8_plane(xrow, c * 8, s.cin - ci0, vec_x);
      }
    }
    ptx::fence_proxy_async();                          // generic-proxy stores -> visible to the wgmma (async proxy)
    __syncthreads();
    wg::fence();
#pragma unroll
    for (int ks = 0; ks < kWgK / 16; ++ks) {
      const uint32_t koff = ks * 16 * 128;
      if constexpr (OP != 0) {
        wg::mma_plane_mn64<OP>(stage, wg::desc_mn_sw128(s_base + 0 * kWgTileBytes + koff, 1024),
                               wg::desc_mn_sw128(s_base + 1 * kWgTileBytes + koff, 1024), ks > 0);
        continue;
      }
      const uint64_t a_hi = wg::desc_mn_sw128(s_base + 0 * kWgTileBytes + koff, 1024);
      const uint64_t a_lo = wg::desc_mn_sw128(s_base + 1 * kWgTileBytes + koff, 1024);
      const uint64_t b_hi = wg::desc_mn_sw128(s_base + 2 * kWgTileBytes + koff, 1024);
      const uint64_t b_lo = wg::desc_mn_sw128(s_base + 3 * kWgTileBytes + koff, 1024);
      wg::mma_bf16_mn64(stage, a_hi, b_hi, ks > 0);
      wg::mma_bf16_mn64(stage, a_hi, b_lo, 1);
      wg::mma_bf16_mn64(stage, a_lo, b_hi, 1);
    }
    wg::commit();
    wg::wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] += stage[i];
    __syncthreads();                                   // every warp's MMAs have read the stage before it is rewritten
  }
  // part[split][tap][co][ci]; accumulator fragment: row = co, column = ci (wgmma.cuh)
  float* dst = part + ((size_t)blockIdx.x * s.kt * s.kh * s.kw + tap) * (size_t)s.cout * s.cin;
  const int w = tid >> 5, l = tid & 31;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int co = co0 + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1);
    const int ci = ci0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    if (co < s.cout && ci < s.cin) dst[(size_t)co * s.cin + ci] = acc[i];
  }
}

// dw[co][ci][ky][kx] = sum over splits (in order) of part[split][tap][co][ci]
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int n_split, int ntaps, int cout, int cin,
                                    float* __restrict__ dw) {
  const size_t n = (size_t)ntaps * cout * cin;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // i enumerates the output layout (co, ci, tap)
  const int tap = (int)(i % ntaps);
  const size_t r = i / ntaps;
  const int ci = (int)(r % cin), co = (int)(r / cin);
  const size_t src = ((size_t)tap * cout + co) * cin + ci;
  float acc = 0.f;
  for (int k = 0; k < n_split; ++k) acc += part[(size_t)k * n + src];
  dw[i] = acc;
}

// ------------------------------------------------------------------------------------------------ channel reductions
// Per-channel sums over n_pix rows, deterministic: grid (channel tiles of 32, kRedParts row ranges, images), block
// (32, 8); fp64 accumulation; partials [image][part][C] to scratch, then one thread per channel adds the parts in order.
// grid.z > 1 (mode 0 only) sums each of gridDim.z consecutive images of n_pix rows on its own.
constexpr int kRedParts = 128;

inline int red_parts(long long n_pix) { return (int)(n_pix < kRedParts ? n_pix : kRedParts); }

// Loaders of `a`: fp32 rows, or bf16 hi/lo rows read as hi + lo (stp3_spatial_sum_det).  a + n moves both.
struct HiLoRows {
  const __nv_bfloat16* hi;
  const __nv_bfloat16* lo;
  __device__ float operator[](long long i) const { return __bfloat162float(hi[i]) + __bfloat162float(lo[i]); }
  __device__ HiLoRows& operator+=(long long n) { hi += n; lo += n; return *this; }
};

// mode 0: sum x;  mode 1: sum (x - mean)^2;  mode 2: sum g' and sum g' * xhat (two outputs), g' = g masked by y > 0
// when y is given, xhat = (x - mean) * invstd (x may be NULL in mode 2: only sum g')
template <class Rows>
__global__ void __launch_bounds__(256)
chan_partial_kernel(int mode, Rows a, int a_cs, const float* __restrict__ y, int y_cs,
                    const float* __restrict__ x, int x_cs, const float* __restrict__ mean,
                    const float* __restrict__ invstd, long long n_pix, int C, double* __restrict__ part) {
  __shared__ double red[2][8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int n_part = gridDim.y;
  a += (long long)blockIdx.z * n_pix * a_cs;
  part += (size_t)blockIdx.z * n_part * 2 * C;
  const long long per = (n_pix + n_part - 1) / n_part;
  const long long p0 = blockIdx.y * per, p1 = p0 + per < n_pix ? p0 + per : n_pix;
  double s0 = 0.0, s1 = 0.0;
  if (c < C) {
    const float m = mean ? mean[c] : 0.f;
    const float is = invstd ? invstd[c] : 0.f;
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const float v = a[p * a_cs + c];
      if (mode == 0) {
        s0 += v;
      } else if (mode == 1) {
        const double d = (double)v - (double)m;
        s0 += d * d;
      } else {
        const float gv = (y && !(y[p * y_cs + c] > 0.f)) ? 0.f : v;
        s0 += gv;
        if (x) s1 += (double)gv * (double)((x[p * x_cs + c] - m) * is);
      }
    }
  }
  red[0][threadIdx.y][threadIdx.x] = s0;
  red[1][threadIdx.y][threadIdx.x] = s1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t0 = 0.0, t1 = 0.0;
    for (int k = 0; k < 8; ++k) { t0 += red[0][k][threadIdx.x]; t1 += red[1][k][threadIdx.x]; }
    part[((size_t)blockIdx.y * 2 + 0) * C + c] = t0;
    part[((size_t)blockIdx.y * 2 + 1) * C + c] = t1;
  }
}

__device__ __forceinline__ void sum_parts(const double* part, int n_part, int C, int c, double& t0, double& t1) {
  t0 = 0.0; t1 = 0.0;
  for (int k = 0; k < n_part; ++k) { t0 += part[((size_t)k * 2) * C + c]; t1 += part[((size_t)k * 2 + 1) * C + c]; }
}

__global__ void mean_finalize_kernel(const double* __restrict__ part, int n_part, int C, long long n_pix,
                                     float* __restrict__ mean) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  mean[c] = (float)(t0 / (double)n_pix);
}

// running = (1 - momentum) * running + momentum * batch, with the roundings spelled out so that every kernel that
// updates running statistics gives the same bits (these are the ones var_finalize_kernel has always produced)
__device__ __forceinline__ void running_update(float* run_mean, float* run_var, int c, float momentum, float mean,
                                               float unb) {
  run_mean[c] = __fmaf_rn(run_mean[c], 1.f - momentum, __fmul_rn(mean, momentum));
  run_var[c] = __fmaf_rn(unb, momentum, __fmul_rn(1.f - momentum, run_var[c]));
}

// biased variance, 1/sqrt(var + eps), and the running statistics (unbiased variance, n / (n - 1)) as nn.BatchNorm2d
__global__ void var_finalize_kernel(const double* __restrict__ part, int n_part, int C, long long n_pix, float eps,
                                    float momentum, const float* __restrict__ mean, float* __restrict__ var,
                                    float* __restrict__ invstd, float* __restrict__ run_mean, float* __restrict__ run_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  const double v = t0 / (double)n_pix;
  if (var) var[c] = (float)v;
  invstd[c] = (float)(1.0 / sqrt(v + (double)eps));
  if (run_mean) {
    const double unb = n_pix > 1 ? v * (double)n_pix / (double)(n_pix - 1) : v;
    running_update(run_mean, run_var, c, momentum, mean[c], (float)unb);
  }
}

// ---- SyncBatchNorm: per-rank fp64 records, merged in rank order (DESIGN.md 3.12)
// A moments record is (4, C) fp64: rows n, S = sum x, Q = sum (x - m)^2, m = the fp32-rounded local mean.  Between the
// two passes row 2 holds m as fp32 (the float the centred pass reads); the second finalize then overwrites it with Q.
__global__ void moments_mean_kernel(const double* __restrict__ part, int n_part, int C, long long n_pix,
                                    double* __restrict__ rec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  const float m = (float)(t0 / (double)n_pix);                   // mean_finalize_kernel's value
  rec[c] = (double)n_pix;
  rec[C + c] = t0;
  rec[3 * C + c] = (double)m;
  reinterpret_cast<float*>(rec + 2 * C)[c] = m;
}

__global__ void moments_q_kernel(const double* __restrict__ part, int n_part, int C, double* __restrict__ rec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  rec[2 * C + c] = t0;
}

// N = sum n_r, mu = sum S_r / N, M2 = sum_r Q_r - 2 d_r (S_r - n_r m_r) + n_r d_r^2 with d_r = mu - m_r (exact algebra:
// sum (x - mu)^2 over rank r's rows, from its centred sum about m_r), in fp64 and rank order.  One record keeps d = 0:
// the variance about the fp32 mean that stp3_bn_stats computes, bit for bit.  The outputs and the running statistics
// are var_finalize_kernel's.
__global__ void bn_merge_finalize_kernel(const double* __restrict__ rec, int world, int C, float eps, float momentum,
                                         float* __restrict__ run_mean, float* __restrict__ run_var,
                                         float* __restrict__ mean, float* __restrict__ var, float* __restrict__ invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double n = 0.0, s = 0.0;
  for (int r = 0; r < world; ++r) { n += rec[(4 * r) * C + c]; s += rec[(4 * r + 1) * C + c]; }
  const double mu = s / n;
  double m2 = 0.0;
  for (int r = 0; r < world; ++r) {
    const double nr = rec[(4 * r) * C + c], sr = rec[(4 * r + 1) * C + c], qr = rec[(4 * r + 2) * C + c];
    const double mr = rec[(4 * r + 3) * C + c];
    const double d = world == 1 ? 0.0 : mu - mr;
    m2 += qr - 2.0 * d * (sr - nr * mr) + nr * d * d;
  }
  const float mf = (float)mu;
  mean[c] = mf;
  const double v = m2 / n;
  if (var) var[c] = (float)v;
  invstd[c] = (float)(1.0 / sqrt(v + (double)eps));
  if (run_mean) {
    const double unb = n > 1.0 ? v * n / (n - 1.0) : v;
    running_update(run_mean, run_var, c, momentum, mf, (float)unb);
  }
}

// backward record (2, C) fp64: sum g', sum g' xhat over this rank's rows
__global__ void sums_record_kernel(const double* __restrict__ part, int n_part, int C, double* __restrict__ rec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  rec[c] = t0;
  rec[C + c] = t1;
}

__global__ void sums_merge_kernel(const double* __restrict__ rec, int world, int C, float* __restrict__ sum_g,
                                  float* __restrict__ sum_gx) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double t0 = 0.0, t1 = 0.0;
  for (int r = 0; r < world; ++r) { t0 += rec[(2 * r) * C + c]; t1 += rec[(2 * r + 1) * C + c]; }
  sum_g[c] = (float)t0;
  sum_gx[c] = (float)t1;
}

// grid.y = images: image i reads its own partials and writes sum_g[i * C + c]
__global__ void sums_finalize_kernel(const double* __restrict__ part, int n_part, int C, float* __restrict__ sum_g,
                                     float* __restrict__ sum_gx) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  part += (size_t)blockIdx.y * n_part * 2 * C;
  sum_g += (size_t)blockIdx.y * C;
  double t0, t1;
  sum_parts(part, n_part, C, c, t0, t1);
  sum_g[c] = (float)t0;
  if (sum_gx) sum_gx[c] = (float)t1;
}

// ------------------------------------------------------------------------------------------------ elementwise
// Philox-4x32-10 (Salmon et al., SC'11): four 32-bit words of counter-based random output for (key, counter)
__device__ __forceinline__ uint4 philox4x32_10(uint32_t k0, uint32_t k1, uint4 c) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// dropout keep bits of the 8 flat elements e0 .. e0 + 7: element e keeps when word e % 4 of
// philox(key = seed, counter = e / 4), read as a 24-bit uniform u in [0, 1), has u >= p
__device__ __forceinline__ uint32_t dropout_keep8(unsigned long long seed, unsigned long long e0, float p) {
  uint32_t bits = 0;
  uint4 r = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const unsigned long long e = e0 + k;
    if (k == 0 || (e & 3) == 0) {
      const unsigned long long q = e >> 2;
      r = philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), make_uint4((uint32_t)q, (uint32_t)(q >> 32), 0u, 0u));
    }
    const uint32_t w = (e & 3) == 0 ? r.x : (e & 3) == 1 ? r.y : (e & 3) == 2 ? r.z : r.w;
    if ((float)(w >> 8) * (1.f / 16777216.f) >= p) bits |= 1u << k;
  }
  return bits;
}

// y = relu?((x - mean) * invstd * gamma + beta (+ res)) [* keep / (1 - p)]; one thread = one pixel x 8 channels (two
// 128-bit loads); groups of 8 channels in [C, y_cs) of the bf16 planes are written as zeros (padding of the next conv's
// K blocks).  Dropout (p > 0): the keep bit of element (pixel, c) depends only on (seed, offset + pixel * C + c).
// OP != 0 (stp3_bn_apply_plane): yh receives ONE bf16 (1) / fp16 (2) plane instead of the hi/lo pair
template <int OP>
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ x, int x_cs, const float* __restrict__ mean, const float* __restrict__ invstd,
                const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ res, int res_cs,
                int relu, float drop_p, unsigned long long seed, unsigned long long offset, long long n_pix, int C,
                float* __restrict__ y, int y_cs, __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl,
                int hl_cs) {
  const int groups = (hl_cs > C ? hl_cs : C) / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * groups) return;
  const int g = (int)(i % groups);
  const long long p = i / groups;
  const int c0 = g * 8;
  float v[8];
  if (c0 < C) {
    const float4 a = *reinterpret_cast<const float4*>(x + p * x_cs + c0);
    const float4 b = *reinterpret_cast<const float4*>(x + p * x_cs + c0 + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    float r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (res) {
      const float4 ra = *reinterpret_cast<const float4*>(res + p * res_cs + c0);
      const float4 rb = *reinterpret_cast<const float4*>(res + p * res_cs + c0 + 4);
      r[0] = ra.x; r[1] = ra.y; r[2] = ra.z; r[3] = ra.w; r[4] = rb.x; r[5] = rb.y; r[6] = rb.z; r[7] = rb.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = c0 + k;
      float t = (v[k] - mean[c]) * invstd[c] * gamma[c] + beta[c] + r[k];
      v[k] = relu ? fmaxf(t, 0.f) : t;
    }
    if (drop_p > 0.f) {
      const uint32_t keep = dropout_keep8(seed, offset + (unsigned long long)p * C + c0, drop_p);
      const float scale = 1.f / (1.f - drop_p);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = (keep >> k) & 1u ? v[k] * scale : 0.f;
    }
    if (y) {
      *reinterpret_cast<float4*>(y + p * y_cs + c0) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(y + p * y_cs + c0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
  }
  if (yh && c0 < hl_cs) {
    if constexpr (OP == 0) {
      uint32_t oh[4], ol[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) ptx::split_hilo(v[2 * e], v[2 * e + 1], oh[e], ol[e]);
      *reinterpret_cast<uint4*>(yh + p * hl_cs + c0) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
      *reinterpret_cast<uint4*>(yl + p * hl_cs + c0) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    } else {
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = ptx::pack_plane16x2<OP>(v[2 * e], v[2 * e + 1]);
      *reinterpret_cast<uint4*>(yh + p * hl_cs + c0) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// dx = gamma * invstd * (g' - sum_g / n - xhat * sum_gx / n) over n_pix rows, n = n_norm (the rows the statistics and
// sums cover: n_pix, or the process group's count under SyncBatchNorm), g' = g masked by y > 0 when y is given; g' is
// also written to gm (the gradient of the residual branch) when gm is given
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ g, int g_cs, const float* __restrict__ y, int y_cs,
                    const float* __restrict__ x, int x_cs, const float* __restrict__ mean, const float* __restrict__ invstd,
                    const float* __restrict__ gamma, const float* __restrict__ sum_g, const float* __restrict__ sum_gx,
                    long long n_pix, long long n_norm, int C, float* __restrict__ dx, int dx_cs, float* __restrict__ gm,
                    int gm_cs) {
  const int groups = C / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * groups) return;
  const int c0 = (int)(i % groups) * 8;
  const long long p = i / groups;
  const float inv_n = 1.f / (float)n_norm;
  float gv[8], xv[8], yv[8];
  auto ld8 = [&](const float* src, float* dst) {
    const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
    dst[0] = a.x; dst[1] = a.y; dst[2] = a.z; dst[3] = a.w; dst[4] = b.x; dst[5] = b.y; dst[6] = b.z; dst[7] = b.w;
  };
  ld8(g + p * g_cs + c0, gv);
  ld8(x + p * x_cs + c0, xv);
  if (y) {
    ld8(y + p * y_cs + c0, yv);
#pragma unroll
    for (int k = 0; k < 8; ++k) if (!(yv[k] > 0.f)) gv[k] = 0.f;
  }
  float o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = c0 + k;
    const float xh = (xv[k] - mean[c]) * invstd[c];
    o[k] = gamma[c] * invstd[c] * (gv[k] - sum_g[c] * inv_n - xh * sum_gx[c] * inv_n);
  }
  *reinterpret_cast<float4*>(dx + p * dx_cs + c0) = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(dx + p * dx_cs + c0 + 4) = make_float4(o[4], o[5], o[6], o[7]);
  if (gm) {
    *reinterpret_cast<float4*>(gm + p * gm_cs + c0) = make_float4(gv[0], gv[1], gv[2], gv[3]);
    *reinterpret_cast<float4*>(gm + p * gm_cs + c0 + 4) = make_float4(gv[4], gv[5], gv[6], gv[7]);
  }
}

// keep bit of one flat element e (the bit dropout_keep8 gives it)
__device__ __forceinline__ bool dropout_keep1(unsigned long long seed, unsigned long long e, float p) {
  const unsigned long long q = e >> 2;
  const uint4 r = philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), make_uint4((uint32_t)q, (uint32_t)(q >> 32), 0u, 0u));
  const uint32_t w = (e & 3) == 0 ? r.x : (e & 3) == 1 ? r.y : (e & 3) == 2 ? r.z : r.w;
  return (float)(w >> 8) * (1.f / 16777216.f) >= p;
}

// bn_apply_kernel for any C and row stride (channel windows at odd offsets, C % 8 != 0): one thread = one element of
// the n_cols = max(C, hl_cs) columns; the same arithmetic per element as the vector kernel
template <int OP>
__global__ void __launch_bounds__(256)
bn_apply_scalar_kernel(const float* __restrict__ x, int x_cs, const float* __restrict__ mean,
                       const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                       const float* __restrict__ res, int res_cs, int relu, float drop_p, unsigned long long seed,
                       unsigned long long offset, long long n_pix, int C, int n_cols, float* __restrict__ y, int y_cs,
                       __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int hl_cs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * n_cols) return;
  const int c = (int)(i % n_cols);
  const long long p = i / n_cols;
  float v = 0.f;
  if (c < C) {
    const float r = res ? res[p * res_cs + c] : 0.f;
    const float t = (x[p * x_cs + c] - mean[c]) * invstd[c] * gamma[c] + beta[c] + r;
    v = relu ? fmaxf(t, 0.f) : t;
    if (drop_p > 0.f) v = dropout_keep1(seed, offset + (unsigned long long)p * C + c, drop_p) ? v * (1.f / (1.f - drop_p)) : 0.f;
    if (y) y[p * y_cs + c] = v;
  }
  if constexpr (OP == 0) {
    if (yh && c < hl_cs) ptx::split_hilo(v, yh[p * hl_cs + c], yl[p * hl_cs + c]);
  } else {
    if (yh && c < hl_cs) reinterpret_cast<uint16_t*>(yh)[p * hl_cs + c] = ptx::plane16<OP>(v);
  }
}

// bn_bwd_apply_kernel for any C and row stride: one thread = one element
__global__ void __launch_bounds__(256)
bn_bwd_apply_scalar_kernel(const float* __restrict__ g, int g_cs, const float* __restrict__ y, int y_cs,
                           const float* __restrict__ x, int x_cs, const float* __restrict__ mean,
                           const float* __restrict__ invstd, const float* __restrict__ gamma,
                           const float* __restrict__ sum_g, const float* __restrict__ sum_gx, long long n_pix,
                           long long n_norm, int C, float* __restrict__ dx, int dx_cs, float* __restrict__ gm, int gm_cs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * C) return;
  const int c = (int)(i % C);
  const long long p = i / C;
  const float inv_n = 1.f / (float)n_norm;
  float gv = g[p * g_cs + c];
  if (y && !(y[p * y_cs + c] > 0.f)) gv = 0.f;
  const float xh = (x[p * x_cs + c] - mean[c]) * invstd[c];
  dx[p * dx_cs + c] = gamma[c] * invstd[c] * (gv - sum_g[c] * inv_n - xh * sum_gx[c] * inv_n);
  if (gm) gm[p * gm_cs + c] = gv;
}

// The pooled branch of a TemporalBlock in time (AvgPool3d((2, H, W)), time padding 1, count_include_pad=False) on
// per-image means m (B, T, C): the T + 1 pooled frames p (B, T + 1, C), p[0] = m[0], p[t] = (m[t-1] + m[t]) / 2 for
// 1 <= t < T, p[T] = m[T-1] (the reference drops that frame only after its BatchNorm).  adjoint: g (B, T + 1, C) ->
// (B, T, C), out[t] = c_t g[t] + (t + 1 < T ? g[t+1] / 2 : g[T]), c_0 = 1, c_t = 1/2.  One thread per output element.
__global__ void __launch_bounds__(256)
temporal_pair_mean_kernel(const float* __restrict__ m, int T, int C, long long total, int adjoint,
                          float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  if (!adjoint) {                                      // i over (B, T + 1, C)
    const int t = (int)(i / C % (T + 1));
    const long long b = i / C / (T + 1);
    const float* mb = m + b * T * C + c;
    out[i] = t == 0 ? mb[0] : t == T ? mb[(long long)(T - 1) * C] : 0.5f * (mb[(long long)(t - 1) * C] + mb[(long long)t * C]);
  } else {                                             // i over (B, T, C)
    const int t = (int)(i / C % T);
    const long long b = i / C / T;
    const float* gb = m + b * (T + 1) * C + c;
    const float a = t == 0 ? gb[0] : 0.5f * gb[(long long)t * C];
    out[i] = a + (t + 1 < T ? 0.5f * gb[(long long)(t + 1) * C] : gb[(long long)T * C]);
  }
}

// bilinear x2, align_corners=False (nn.Upsample of UpsamplingAdd): source coordinate (o + 0.5) / 2 - 0.5 clamped at 0
__device__ __forceinline__ void up_coord(int o, int n, int& i0, int& i1, float& w0, float& w1) {
  const float f = fmaxf((o + 0.5f) * 0.5f - 0.5f, 0.f);
  i0 = (int)f;
  i1 = min(i0 + 1, n - 1);
  w1 = f - i0;
  w0 = 1.f - w1;
}

// V consecutive fp32 channels (V = 4: one 16-byte access; V = 1: any alignment)
template <int V>
__device__ __forceinline__ void ld_vec(const float* p, float (&v)[V]) {
  if constexpr (V == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = *p;
  }
}
template <int V>
__device__ __forceinline__ void st_vec(float* p, const float (&v)[V]) {
  if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else *p = v[0];
}

// y[.., y_coff + c] = bilinear_x2(x (n_img, h, w, C))[.., c]: y has rows of y_cstride floats (a channel window of a wider
// channels-last tensor, or y_cstride = C, y_coff = 0 for a dense one); one thread per V channels of an output pixel
template <int V>
__global__ void __launch_bounds__(256)
upsample2x_f32_kernel(const float* __restrict__ x, int h, int w, int C, long long total, float* __restrict__ y,
                      int y_cstride, int y_coff) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % (C / V)) * V;
  long long r = i / (C / V);
  const int ox = (int)(r % (2 * w));
  const long long orow = r;                         // output pixel index (img, oy, ox)
  r /= 2 * w;
  const int oy = (int)(r % (2 * h));
  const long long img = r / (2 * h);
  int y0, y1, x0, x1;
  float wy0, wy1, wx0, wx1;
  up_coord(oy, h, y0, y1, wy0, wy1);
  up_coord(ox, w, x0, x1, wx0, wx1);
  const float* b = x + img * h * w * C + c;
  float v00[V], v01[V], v10[V], v11[V], v[V];
  ld_vec<V>(b + ((long long)y0 * w + x0) * C, v00);
  ld_vec<V>(b + ((long long)y0 * w + x1) * C, v01);
  ld_vec<V>(b + ((long long)y1 * w + x0) * C, v10);
  ld_vec<V>(b + ((long long)y1 * w + x1) * C, v11);
#pragma unroll
  for (int k = 0; k < V; ++k) v[k] = wy0 * (wx0 * v00[k] + wx1 * v01[k]) + wy1 * (wx0 * v10[k] + wx1 * v11[k]);
  st_vec<V>(y + orow * y_cstride + y_coff + c, v);
}

// weight of low-resolution index i in output o along one axis (both corners may coincide at the border)
__device__ __forceinline__ float up_weight(int o, int n, int i) {
  int i0, i1;
  float w0, w1;
  up_coord(o, n, i0, i1, w0, w1);
  return (i0 == i ? w0 : 0.f) + (i1 == i ? w1 : 0.f);
}

// gx (n_img, h, w, C) = adjoint of bilinear_x2 applied to channels [gy_coff, gy_coff + C) of gy (n_img, 2h, 2w,
// gy_cstride): a gather over the outputs 2i-1 .. 2i+2 of every axis (fixed order, no atomics)
template <int V>
__global__ void __launch_bounds__(256)
upsample2x_bwd_kernel(const float* __restrict__ gy, int gy_cstride, int gy_coff, int h, int w, int C, long long total,
                      float* __restrict__ gx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % (C / V)) * V;
  long long r = i / (C / V);
  const int ix = (int)(r % w); r /= w;
  const int iy = (int)(r % h);
  const long long img = r / h;
  const float* b = gy + img * 4 * h * w * gy_cstride + gy_coff + c;
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  for (int oy = 2 * iy - 1; oy <= 2 * iy + 2; ++oy) {
    if (oy < 0 || oy >= 2 * h) continue;
    const float wy = up_weight(oy, h, iy);
    if (wy == 0.f) continue;
    float row[V];
#pragma unroll
    for (int k = 0; k < V; ++k) row[k] = 0.f;
    for (int ox = 2 * ix - 1; ox <= 2 * ix + 2; ++ox) {
      if (ox < 0 || ox >= 2 * w) continue;
      const float wx = up_weight(ox, w, ix);
      if (wx != 0.f) {
        float g[V];
        ld_vec<V>(b + ((long long)oy * 2 * w + ox) * gy_cstride, g);
#pragma unroll
        for (int k = 0; k < V; ++k) row[k] = fmaf(wx, g[k], row[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] = fmaf(wy, row[k], acc[k]);
  }
  st_vec<V>(gx + i * V, acc);                       // gx is dense: thread i owns its elements [i * V, i * V + V)
}

// out (n_img, H, W, C)[y][x] = phase[y % 2][x % 2] (n_img, (H - y%2 + 1) / 2, (W - x%2 + 1) / 2, C)[y / 2][x / 2]
// (NULL phase = zeros)
struct Phases { const float* p[4]; };
__global__ void __launch_bounds__(256)
phase_interleave_kernel(Phases ph, int H, int W, int C, long long total, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  long long r = i / C;
  const int x = (int)(r % W); r /= W;
  const int y = (int)(r % H);
  const long long img = r / H;
  const int py = y & 1, px = x & 1;
  const float* src = py ? (px ? ph.p[3] : ph.p[2]) : (px ? ph.p[1] : ph.p[0]);
  float v = 0.f;
  if (src) {
    const int Hp = (H - py + 1) / 2, Wp = (W - px + 1) / 2;
    v = src[((img * Hp + y / 2) * Wp + x / 2) * C + c];
  }
  out[i] = v;
}

// dz = g * s * (1 - s) where s = sigmoid(z) is the forward output
__global__ void sigmoid_bwd_kernel(const float* __restrict__ g, const float* __restrict__ s, long long n,
                                   float* __restrict__ dz) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = s[i];
  dz[i] = g[i] * v * (1.f - v);
}

inline unsigned blocks_for(long long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace stp3

using namespace stp3;

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" size_t stp3_conv_wgrad_scratch_bytes(int n_img, int Ho, int Wo, int cout, int cin, int kh, int kw,
                                                int dilation) {
  if (n_img <= 0 || Ho <= 0 || Wo <= 0 || cout <= 0 || cin <= 0 || kh <= 0 || kw <= 0 || dilation < 1) return 0;
  WgradShape s{};
  s.n_img = n_img; s.Ho = Ho; s.Wo = Wo; s.cout = cout; s.cin = cin; s.kh = kh; s.kw = kw;
  return (size_t)wgrad_splits(s) * kh * kw * (size_t)cout * cin * sizeof(float);
}

// the partial GEMMs and the ordered reduction of one (validated) weight gradient (OP: operand kind, STP3_OPERAND_*)
template <int OP = 0, typename In = float>
static int launch_wgrad(const WgradShape& s, const In* x, const In* g, float* scratch, float* dw, cudaStream_t st,
                        const char* what) {
  const int n_split = wgrad_splits(s);
  const long long P = wgrad_pixels(s);
  long long per = (P + n_split - 1) / n_split;
  per = (per + kWgK - 1) / kWgK * kWgK;
  const int ntaps = s.kt * s.kh * s.kw;
  const long long tiles = (long long)ntaps * ceil_div(s.cout, kWgTile) * ceil_div(s.cin, kWgTile);
  if (tiles >= 65536) return stp3::set_error(STP3_EINVAL, "%s: too many output tiles", what);
  // 16-byte loads need 16-byte aligned rows
  constexpr int kPerChunk = 16 / sizeof(In);
  const int vec_x = s.x_cstride % kPerChunk == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const int vec_g = s.g_cstride % kPerChunk == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const size_t smem = (OP == 0 ? 4 : 2) * kWgTileBytes + 1024;
  wgrad_partial_kernel<OP><<<dim3(n_split, (unsigned)tiles), 128, smem, st>>>(x, g, s, per, vec_x, vec_g, scratch);
  STP3_CUDA_OK(cudaGetLastError());
  const long long n = (long long)ntaps * s.cout * s.cin;
  wgrad_reduce_kernel<<<blocks_for(n), 256, 0, st>>>(scratch, n_split, ntaps, s.cout, s.cin, dw);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_conv_wgrad(const float* x, int n_img, int H, int W, int x_cstride, int cin, const float* g, int Ho,
                               int Wo, int g_cstride, int cout, int kh, int kw, int stride, int pad, int dilation,
                               void* scratch, size_t scratch_bytes, float* dw, void* stream) {
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_conv_wgrad: null pointer argument");
  STP3_CHECK_ARG(n_img > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && cin > 0 && cout > 0 && kh > 0 && kw > 0 && pad >= 0,
                 "stp3_conv_wgrad: non-positive dimension");
  STP3_CHECK_ARG(stride == 1 || stride == 2, "stp3_conv_wgrad: stride must be 1 or 2");
  STP3_CHECK_ARG(dilation >= 1, "stp3_conv_wgrad: dilation must be >= 1");
  STP3_CHECK_ARG(cin <= x_cstride && cout <= g_cstride, "stp3_conv_wgrad: channel count exceeds the row stride");
  const size_t need = stp3_conv_wgrad_scratch_bytes(n_img, Ho, Wo, cout, cin, kh, kw, dilation);
  STP3_CHECK_ARG(scratch_bytes >= need, "stp3_conv_wgrad: scratch smaller than stp3_conv_wgrad_scratch_bytes()");
  WgradShape s{n_img, H, W, x_cstride, cin, Ho, Wo, g_cstride, cout, stride, kh, kw, pad, dilation};
  return launch_wgrad(s, x, g, (float*)scratch, dw, (cudaStream_t)stream, "stp3_conv_wgrad");
}

extern "C" size_t stp3_conv3d_wgrad_scratch_bytes(int B, int T, int H, int W, int cout, int cin, int kt, int kh, int kw) {
  if (B <= 0 || T <= 0 || H <= 0 || W <= 0 || cout <= 0 || cin <= 0 || kt <= 0 || kh <= 0 || kw <= 0) return 0;
  if ((long long)B * T > INT_MAX) return 0;
  WgradShape s{};
  s.n_img = B * T; s.Ho = H; s.Wo = W; s.cout = cout; s.cin = cin; s.kh = kh; s.kw = kw; s.T = T; s.kt = kt;
  return (size_t)wgrad_splits(s) * kt * kh * kw * (size_t)cout * cin * sizeof(float);
}

extern "C" int stp3_conv3d_wgrad(const float* x, int B, int T, int H, int W, int x_cstride, int cin, const float* g,
                                 int g_cstride, int cout, int kt, int kh, int kw, void* scratch, size_t scratch_bytes,
                                 float* dw, void* stream) {
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_conv3d_wgrad: null pointer argument");
  STP3_CHECK_ARG(B > 0 && T > 0 && H > 0 && W > 0 && cin > 0 && cout > 0 && kt > 0 && kh > 0 && kw > 0,
                 "stp3_conv3d_wgrad: non-positive dimension");
  STP3_CHECK_ARG((long long)B * T <= INT_MAX, "stp3_conv3d_wgrad: too many frames");
  STP3_CHECK_ARG(kh == kw && kh % 2 == 1, "stp3_conv3d_wgrad: the spatial kernel must be square and odd");
  STP3_CHECK_ARG(cin <= x_cstride && cout <= g_cstride, "stp3_conv3d_wgrad: channel count exceeds the row stride");
  const size_t need = stp3_conv3d_wgrad_scratch_bytes(B, T, H, W, cout, cin, kt, kh, kw);
  STP3_CHECK_ARG(scratch_bytes >= need, "stp3_conv3d_wgrad: scratch smaller than stp3_conv3d_wgrad_scratch_bytes()");
  WgradShape s{B * T, H, W, x_cstride, cin, H, W, g_cstride, cout, 1, kh, kw, (kh - 1) / 2, 1};
  s.T = T; s.kt = kt;
  return launch_wgrad(s, x, g, (float*)scratch, dw, (cudaStream_t)stream, "stp3_conv3d_wgrad");
}

static int launch_wgrad_plane(int operand, const WgradShape& s, const void* x, const void* g, void* scratch, float* dw,
                              void* stream, const char* what) {
  const uint16_t* xs = static_cast<const uint16_t*>(x);
  const uint16_t* gs = static_cast<const uint16_t*>(g);
  if (operand == STP3_OPERAND_F16)
    return launch_wgrad<STP3_OPERAND_F16>(s, xs, gs, (float*)scratch, dw, (cudaStream_t)stream, what);
  return launch_wgrad<STP3_OPERAND_BF16>(s, xs, gs, (float*)scratch, dw, (cudaStream_t)stream, what);
}

extern "C" int stp3_conv_wgrad_plane(int operand, const void* x, int n_img, int H, int W, int x_cstride, int cin,
                                     const void* g, int Ho, int Wo, int g_cstride, int cout, int kh, int kw, int stride,
                                     int pad, int dilation, void* scratch, size_t scratch_bytes, float* dw,
                                     void* stream) {
  STP3_CHECK_ARG(operand == STP3_OPERAND_BF16 || operand == STP3_OPERAND_F16,
                 "stp3_conv_wgrad_plane: operand must be STP3_OPERAND_BF16 or STP3_OPERAND_F16");
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_conv_wgrad_plane: null pointer argument");
  STP3_CHECK_ARG(n_img > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && cin > 0 && cout > 0 && kh > 0 && kw > 0 && pad >= 0,
                 "stp3_conv_wgrad_plane: non-positive dimension");
  STP3_CHECK_ARG(stride == 1 || stride == 2, "stp3_conv_wgrad_plane: stride must be 1 or 2");
  STP3_CHECK_ARG(dilation >= 1, "stp3_conv_wgrad_plane: dilation must be >= 1");
  STP3_CHECK_ARG(cin <= x_cstride && cout <= g_cstride, "stp3_conv_wgrad_plane: channel count exceeds the row stride");
  const size_t need = stp3_conv_wgrad_scratch_bytes(n_img, Ho, Wo, cout, cin, kh, kw, dilation);
  STP3_CHECK_ARG(scratch_bytes >= need, "stp3_conv_wgrad_plane: scratch smaller than stp3_conv_wgrad_scratch_bytes()");
  WgradShape s{n_img, H, W, x_cstride, cin, Ho, Wo, g_cstride, cout, stride, kh, kw, pad, dilation};
  return launch_wgrad_plane(operand, s, x, g, scratch, dw, stream, "stp3_conv_wgrad_plane");
}

extern "C" int stp3_conv3d_wgrad_plane(int operand, const void* x, int B, int T, int H, int W, int x_cstride, int cin,
                                       const void* g, int g_cstride, int cout, int kt, int kh, int kw, void* scratch,
                                       size_t scratch_bytes, float* dw, void* stream) {
  STP3_CHECK_ARG(operand == STP3_OPERAND_BF16 || operand == STP3_OPERAND_F16,
                 "stp3_conv3d_wgrad_plane: operand must be STP3_OPERAND_BF16 or STP3_OPERAND_F16");
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_conv3d_wgrad_plane: null pointer argument");
  STP3_CHECK_ARG(B > 0 && T > 0 && H > 0 && W > 0 && cin > 0 && cout > 0 && kt > 0 && kh > 0 && kw > 0,
                 "stp3_conv3d_wgrad_plane: non-positive dimension");
  STP3_CHECK_ARG((long long)B * T <= INT_MAX, "stp3_conv3d_wgrad_plane: too many frames");
  STP3_CHECK_ARG(kh == kw && kh % 2 == 1, "stp3_conv3d_wgrad_plane: the spatial kernel must be square and odd");
  STP3_CHECK_ARG(cin <= x_cstride && cout <= g_cstride, "stp3_conv3d_wgrad_plane: channel count exceeds the row stride");
  const size_t need = stp3_conv3d_wgrad_scratch_bytes(B, T, H, W, cout, cin, kt, kh, kw);
  STP3_CHECK_ARG(scratch_bytes >= need, "stp3_conv3d_wgrad_plane: scratch smaller than stp3_conv3d_wgrad_scratch_bytes()");
  WgradShape s{B * T, H, W, x_cstride, cin, H, W, g_cstride, cout, 1, kh, kw, (kh - 1) / 2, 1};
  s.T = T; s.kt = kt;
  return launch_wgrad_plane(operand, s, x, g, scratch, dw, stream, "stp3_conv3d_wgrad_plane");
}

extern "C" size_t stp3_bn_scratch_bytes(long long n_pix, int C) {
  if (n_pix <= 0 || C <= 0) return 0;
  return (size_t)red_parts(n_pix) * 2 * C * sizeof(double);
}

extern "C" int stp3_bn_stats(const float* x, long long n_pix, int C, int x_cstride, float eps, float momentum,
                             float* running_mean, float* running_var, float* mean, float* var, float* invstd,
                             void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(x && mean && invstd && scratch && n_pix > 0 && C > 0 && C <= x_cstride, "stp3_bn_stats: bad argument");
  STP3_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr), "stp3_bn_stats: give both running buffers or neither");
  STP3_CHECK_ARG(scratch_bytes >= stp3_bn_scratch_bytes(n_pix, C), "stp3_bn_stats: scratch smaller than stp3_bn_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(n_pix);
  double* part = (double*)scratch;
  const dim3 grid(ceil_div(C, 32), parts), block(32, 8);
  chan_partial_kernel<<<grid, block, 0, st>>>(0, x, x_cstride, nullptr, 0, nullptr, 0, nullptr, nullptr, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  mean_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, n_pix, mean);
  STP3_CUDA_OK(cudaGetLastError());
  chan_partial_kernel<<<grid, block, 0, st>>>(1, x, x_cstride, nullptr, 0, nullptr, 0, mean, nullptr, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  var_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, n_pix, eps, momentum, mean, var, invstd,
                                                         running_mean, running_var);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

// stp3_bn_apply (OP 0: y_hi / y_lo) and stp3_bn_apply_plane (OP 1 / 2: one plane in y_hi, y_lo NULL)
template <int OP>
static int bn_apply(const float* x, long long n_pix, int C, int x_cstride, const float* mean, const float* invstd,
                    const float* gamma, const float* beta, const float* res, int res_cstride, int relu, float dropout_p,
                    unsigned long long seed, unsigned long long offset, float* y, int y_cstride, void* y_hi, void* y_lo,
                    int hl_cstride, void* stream) {
  STP3_CHECK_ARG(x && mean && invstd && gamma && beta && (y || y_hi) && n_pix > 0 && C > 0, "stp3_bn_apply: bad argument");
  STP3_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "stp3_bn_apply: dropout p must be in [0, 1)");
  if (OP == 0) STP3_CHECK_ARG((y_hi == nullptr) == (y_lo == nullptr), "stp3_bn_apply: give both bf16 planes or neither");
  STP3_CHECK_ARG(C <= x_cstride, "stp3_bn_apply: C exceeds the row stride");
  STP3_CHECK_ARG(!res || C <= res_cstride, "stp3_bn_apply: bad residual");
  STP3_CHECK_ARG(!y || C <= y_cstride, "stp3_bn_apply: bad fp32 output");
  STP3_CHECK_ARG(!y_hi || (hl_cstride % 8 == 0 && C <= hl_cstride && al16(y_hi) && (OP != 0 || al16(y_lo))),
                 "stp3_bn_apply: bad bf16 planes");
  // 8 channels per thread with 128-bit accesses when every row allows it, else one element per thread
  const bool vec = C % 8 == 0 && x_cstride % 4 == 0 && al16(x) && (!res || (res_cstride % 4 == 0 && al16(res))) &&
                   (!y || (y_cstride % 4 == 0 && al16(y)));
  if (!vec) {
    const int n_cols = (y_hi && hl_cstride > C) ? hl_cstride : C;
    bn_apply_scalar_kernel<OP><<<blocks_for(n_pix * n_cols), 256, 0, (cudaStream_t)stream>>>(
        x, x_cstride, mean, invstd, gamma, beta, res, res_cstride, relu, dropout_p, seed, offset, n_pix, C, n_cols, y,
        y_cstride, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, y_hi ? hl_cstride : 0);
    STP3_CUDA_OK(cudaGetLastError());
    return STP3_OK;
  }
  const int groups = ((y_hi && hl_cstride > C) ? hl_cstride : C) / 8;
  const long long total = n_pix * groups;
  bn_apply_kernel<OP><<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(
      x, x_cstride, mean, invstd, gamma, beta, res, res_cstride, relu, dropout_p, seed, offset, n_pix, C, y, y_cstride,
      (__nv_bfloat16*)y_hi,
      (__nv_bfloat16*)y_lo, y_hi ? hl_cstride : 0);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_apply(const float* x, long long n_pix, int C, int x_cstride, const float* mean,
                             const float* invstd, const float* gamma, const float* beta, const float* res,
                             int res_cstride, int relu, float dropout_p, unsigned long long seed,
                             unsigned long long offset, float* y, int y_cstride, void* y_hi, void* y_lo, int hl_cstride,
                             void* stream) {
  return bn_apply<0>(x, n_pix, C, x_cstride, mean, invstd, gamma, beta, res, res_cstride, relu, dropout_p, seed, offset,
                     y, y_cstride, y_hi, y_lo, hl_cstride, stream);
}

extern "C" int stp3_bn_apply_plane(const float* x, long long n_pix, int C, int x_cstride, const float* mean,
                                   const float* invstd, const float* gamma, const float* beta, const float* res,
                                   int res_cstride, int relu, float dropout_p, unsigned long long seed,
                                   unsigned long long offset, float* y, int y_cstride, void* y_plane,
                                   int plane_cstride, int operand, void* stream) {
  STP3_CHECK_ARG(operand == STP3_OPERAND_BF16 || operand == STP3_OPERAND_F16,
                 "stp3_bn_apply_plane: operand must be STP3_OPERAND_BF16 or STP3_OPERAND_F16");
  if (operand == STP3_OPERAND_F16)
    return bn_apply<2>(x, n_pix, C, x_cstride, mean, invstd, gamma, beta, res, res_cstride, relu, dropout_p, seed,
                       offset, y, y_cstride, y_plane, nullptr, plane_cstride, stream);
  return bn_apply<1>(x, n_pix, C, x_cstride, mean, invstd, gamma, beta, res, res_cstride, relu, dropout_p, seed, offset,
                     y, y_cstride, y_plane, nullptr, plane_cstride, stream);
}

extern "C" int stp3_bn_bwd_reduce(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                                  int x_cstride, const float* mean, const float* invstd, long long n_pix, int C,
                                  float* sum_g, float* sum_gxhat, void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(g && sum_g && scratch && n_pix > 0 && C > 0 && C <= g_cstride, "stp3_bn_bwd_reduce: bad argument");
  STP3_CHECK_ARG(!x || (mean && invstd && sum_gxhat && C <= x_cstride), "stp3_bn_bwd_reduce: x needs mean, invstd, sum_gxhat");
  STP3_CHECK_ARG(!y || C <= y_cstride, "stp3_bn_bwd_reduce: bad mask tensor");
  STP3_CHECK_ARG(scratch_bytes >= stp3_bn_scratch_bytes(n_pix, C), "stp3_bn_bwd_reduce: scratch smaller than stp3_bn_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(n_pix);
  double* part = (double*)scratch;
  chan_partial_kernel<<<dim3(ceil_div(C, 32), parts), dim3(32, 8), 0, st>>>(2, g, g_cstride, y, y_cstride, x, x_cstride,
                                                                          mean, invstd, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  sums_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, sum_g, x ? sum_gxhat : nullptr);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" size_t stp3_image_channel_sums_scratch_bytes(int n_img, long long hw, int C) {
  if (n_img <= 0) return 0;
  return (size_t)n_img * stp3_bn_scratch_bytes(hw, C);
}

extern "C" int stp3_image_channel_sums(const float* x, int n_img, long long hw, int C, int x_cstride, float* sums,
                                       void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(x && sums && scratch && n_img > 0 && hw > 0 && C > 0 && C <= x_cstride,
                 "stp3_image_channel_sums: bad argument");
  STP3_CHECK_ARG(n_img <= 65535, "stp3_image_channel_sums: more than 65535 images");
  STP3_CHECK_ARG(scratch_bytes >= stp3_image_channel_sums_scratch_bytes(n_img, hw, C),
                 "stp3_image_channel_sums: scratch smaller than stp3_image_channel_sums_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(hw);
  double* part = (double*)scratch;
  chan_partial_kernel<<<dim3(ceil_div(C, 32), parts, n_img), dim3(32, 8), 0, st>>>(0, x, x_cstride, nullptr, 0, nullptr, 0,
                                                                                 nullptr, nullptr, hw, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  sums_finalize_kernel<<<dim3(ceil_div(C, 128), n_img), 128, 0, st>>>(part, parts, C, sums, nullptr);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

// stp3_spatial_sum's result with stp3_image_channel_sums' two passes: every pixel's hi + lo, fp64 partials over fixed
// pixel ranges, added in range order
extern "C" size_t stp3_spatial_sum_det_scratch_bytes(int n_img, int HW, int cstride) {
  if (HW <= 0 || cstride <= 0) return 0;
  return stp3_image_channel_sums_scratch_bytes(n_img, HW, cstride);
}

extern "C" int stp3_spatial_sum_det(const void* hi, const void* lo, int n_img, int HW, int cstride, float* sums,
                                    void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(hi && lo && sums && scratch && n_img > 0 && HW > 0 && cstride > 0 && cstride <= 1024,
                 "stp3_spatial_sum_det: bad argument");
  STP3_CHECK_ARG(n_img <= 65535, "stp3_spatial_sum_det: more than 65535 images");
  STP3_CHECK_ARG(scratch_bytes >= stp3_spatial_sum_det_scratch_bytes(n_img, HW, cstride),
                 "stp3_spatial_sum_det: scratch smaller than stp3_spatial_sum_det_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(HW);
  double* part = (double*)scratch;
  const HiLoRows rows{(const __nv_bfloat16*)hi, (const __nv_bfloat16*)lo};
  chan_partial_kernel<<<dim3(ceil_div(cstride, 32), parts, n_img), dim3(32, 8), 0, st>>>(
      0, rows, cstride, nullptr, 0, nullptr, 0, nullptr, nullptr, HW, cstride, part);
  STP3_CUDA_OK(cudaGetLastError());
  sums_finalize_kernel<<<dim3(ceil_div(cstride, 128), n_img), 128, 0, st>>>(part, parts, cstride, sums, nullptr);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

static int bn_bwd_apply_impl(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                             int x_cstride, const float* mean, const float* invstd, const float* gamma,
                             const float* sum_g, const float* sum_gxhat, long long n_pix, long long n_norm, int C,
                             float* dx, int dx_cstride, float* g_masked, int gm_cstride, void* stream) {
  STP3_CHECK_ARG(g && x && mean && invstd && gamma && sum_g && sum_gxhat && dx && n_pix > 0 && C > 0,
                 "stp3_bn_bwd_apply: bad argument");
  STP3_CHECK_ARG(C <= g_cstride && C <= x_cstride && C <= dx_cstride, "stp3_bn_bwd_apply: C exceeds a row stride");
  STP3_CHECK_ARG(!y || C <= y_cstride, "stp3_bn_bwd_apply: bad mask tensor");
  STP3_CHECK_ARG(!g_masked || C <= gm_cstride, "stp3_bn_bwd_apply: bad g_masked");
  const bool vec = C % 8 == 0 && g_cstride % 4 == 0 && x_cstride % 4 == 0 && dx_cstride % 4 == 0 && al16(g) && al16(x) &&
                   al16(dx) && (!y || (y_cstride % 4 == 0 && al16(y))) &&
                   (!g_masked || (gm_cstride % 4 == 0 && al16(g_masked)));
  if (!vec) {
    bn_bwd_apply_scalar_kernel<<<blocks_for(n_pix * C), 256, 0, (cudaStream_t)stream>>>(
        g, g_cstride, y, y_cstride, x, x_cstride, mean, invstd, gamma, sum_g, sum_gxhat, n_pix, n_norm, C, dx,
        dx_cstride, g_masked, gm_cstride);
    STP3_CUDA_OK(cudaGetLastError());
    return STP3_OK;
  }
  const long long total = n_pix * (C / 8);
  bn_bwd_apply_kernel<<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(
      g, g_cstride, y, y_cstride, x, x_cstride, mean, invstd, gamma, sum_g, sum_gxhat, n_pix, n_norm, C, dx, dx_cstride,
      g_masked, gm_cstride);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_bwd_apply(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                                 int x_cstride, const float* mean, const float* invstd, const float* gamma,
                                 const float* sum_g, const float* sum_gxhat, long long n_pix, int C, float* dx,
                                 int dx_cstride, float* g_masked, int gm_cstride, void* stream) {
  return bn_bwd_apply_impl(g, g_cstride, y, y_cstride, x, x_cstride, mean, invstd, gamma, sum_g, sum_gxhat, n_pix, n_pix,
                           C, dx, dx_cstride, g_masked, gm_cstride, stream);
}

// ------------------------------------------------------------------------------------------------ SyncBatchNorm
extern "C" int stp3_bn_local_moments(const float* x, long long n_pix, int C, int x_cstride, double* out, void* scratch,
                                     size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(x && out && scratch && n_pix > 0 && C > 0 && C <= x_cstride, "stp3_bn_local_moments: bad argument");
  STP3_CHECK_ARG(scratch_bytes >= stp3_bn_scratch_bytes(n_pix, C),
                 "stp3_bn_local_moments: scratch smaller than stp3_bn_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(n_pix);
  double* part = (double*)scratch;
  const dim3 grid(ceil_div(C, 32), parts), block(32, 8);
  chan_partial_kernel<<<grid, block, 0, st>>>(0, x, x_cstride, nullptr, 0, nullptr, 0, nullptr, nullptr, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  moments_mean_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, n_pix, out);
  STP3_CUDA_OK(cudaGetLastError());
  chan_partial_kernel<<<grid, block, 0, st>>>(1, x, x_cstride, nullptr, 0, nullptr, 0,
                                              reinterpret_cast<const float*>(out + 2 * C), nullptr, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  moments_q_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_merge_finalize(const double* records, int world, int C, float eps, float momentum,
                                      float* running_mean, float* running_var, float* mean, float* var, float* invstd,
                                      void* stream) {
  STP3_CHECK_ARG(records && mean && invstd && world > 0 && C > 0, "stp3_bn_merge_finalize: bad argument");
  STP3_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr),
                 "stp3_bn_merge_finalize: give both running buffers or neither");
  bn_merge_finalize_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(records, world, C, eps, momentum,
                                                                               running_mean, running_var, mean, var,
                                                                               invstd);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_bwd_local_sums(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                                      int x_cstride, const float* mean, const float* invstd, long long n_pix, int C,
                                      double* out, void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(g && x && mean && invstd && out && scratch && n_pix > 0 && C > 0 && C <= g_cstride && C <= x_cstride,
                 "stp3_bn_bwd_local_sums: bad argument");
  STP3_CHECK_ARG(!y || C <= y_cstride, "stp3_bn_bwd_local_sums: bad mask tensor");
  STP3_CHECK_ARG(scratch_bytes >= stp3_bn_scratch_bytes(n_pix, C),
                 "stp3_bn_bwd_local_sums: scratch smaller than stp3_bn_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = red_parts(n_pix);
  double* part = (double*)scratch;
  chan_partial_kernel<<<dim3(ceil_div(C, 32), parts), dim3(32, 8), 0, st>>>(2, g, g_cstride, y, y_cstride, x, x_cstride,
                                                                          mean, invstd, n_pix, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  sums_record_kernel<<<ceil_div(C, 128), 128, 0, st>>>(part, parts, C, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_bwd_merge_sums(const double* records, int world, int C, float* sum_g, float* sum_gxhat,
                                      void* stream) {
  STP3_CHECK_ARG(records && sum_g && sum_gxhat && world > 0 && C > 0, "stp3_bn_bwd_merge_sums: bad argument");
  sums_merge_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(records, world, C, sum_g, sum_gxhat);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_bn_bwd_apply_global(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                                        int x_cstride, const float* mean, const float* invstd, const float* gamma,
                                        const float* sum_g, const float* sum_gxhat, long long n_pix, long long n_total,
                                        int C, float* dx, int dx_cstride, float* g_masked, int gm_cstride,
                                        void* stream) {
  STP3_CHECK_ARG(n_total >= n_pix, "stp3_bn_bwd_apply_global: n_total is smaller than n_pix");
  return bn_bwd_apply_impl(g, g_cstride, y, y_cstride, x, x_cstride, mean, invstd, gamma, sum_g, sum_gxhat, n_pix,
                           n_total, C, dx, dx_cstride, g_masked, gm_cstride, stream);
}

// 16-byte accesses when every row of the dense tensor and of the window starts 16-byte aligned; else one float per thread
static bool upsample_vec(const void* dense, const void* win, int C, int cstride, int coff) {
  return C % 4 == 0 && cstride % 4 == 0 && coff % 4 == 0 && reinterpret_cast<uintptr_t>(dense) % 16 == 0 &&
         reinterpret_cast<uintptr_t>(win) % 16 == 0;
}

extern "C" int stp3_upsample2x_window_f32(const float* x, int n_img, int h, int w, int C, float* y, int y_cstride,
                                          int y_coff, void* stream) {
  STP3_CHECK_ARG(x && y && n_img > 0 && h > 0 && w > 0 && C > 0, "stp3_upsample2x_window_f32: bad argument");
  STP3_CHECK_ARG(y_coff >= 0 && y_coff + C <= y_cstride,
                 "stp3_upsample2x_window_f32: channels [%d, %d) outside rows of %d", y_coff, y_coff + C, y_cstride);
  const long long pix = (long long)n_img * 4 * h * w;
  if (upsample_vec(x, y, C, y_cstride, y_coff))
    upsample2x_f32_kernel<4><<<blocks_for(pix * (C / 4)), 256, 0, (cudaStream_t)stream>>>(x, h, w, C, pix * (C / 4), y,
                                                                                         y_cstride, y_coff);
  else
    upsample2x_f32_kernel<1><<<blocks_for(pix * C), 256, 0, (cudaStream_t)stream>>>(x, h, w, C, pix * C, y, y_cstride,
                                                                                   y_coff);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_upsample2x_window_bwd(const float* gy, int gy_cstride, int gy_coff, int n_img, int h, int w, int C,
                                          float* gx, void* stream) {
  STP3_CHECK_ARG(gy && gx && n_img > 0 && h > 0 && w > 0 && C > 0, "stp3_upsample2x_window_bwd: bad argument");
  STP3_CHECK_ARG(gy_coff >= 0 && gy_coff + C <= gy_cstride,
                 "stp3_upsample2x_window_bwd: channels [%d, %d) outside rows of %d", gy_coff, gy_coff + C, gy_cstride);
  const long long pix = (long long)n_img * h * w;
  if (upsample_vec(gx, gy, C, gy_cstride, gy_coff))
    upsample2x_bwd_kernel<4><<<blocks_for(pix * (C / 4)), 256, 0, (cudaStream_t)stream>>>(gy, gy_cstride, gy_coff, h, w,
                                                                                         C, pix * (C / 4), gx);
  else
    upsample2x_bwd_kernel<1><<<blocks_for(pix * C), 256, 0, (cudaStream_t)stream>>>(gy, gy_cstride, gy_coff, h, w, C,
                                                                                   pix * C, gx);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_upsample2x_f32(const float* x, int n_img, int h, int w, int C, float* y, void* stream) {
  STP3_CHECK_ARG(x && y && n_img > 0 && h > 0 && w > 0 && C > 0, "stp3_upsample2x_f32: bad argument");
  return stp3_upsample2x_window_f32(x, n_img, h, w, C, y, C, 0, stream);
}

extern "C" int stp3_upsample2x_bwd(const float* gy, int n_img, int h, int w, int C, float* gx, void* stream) {
  STP3_CHECK_ARG(gy && gx && n_img > 0 && h > 0 && w > 0 && C > 0, "stp3_upsample2x_bwd: bad argument");
  return stp3_upsample2x_window_bwd(gy, C, 0, n_img, h, w, C, gx, stream);
}

extern "C" int stp3_phase_interleave(const float* p00, const float* p01, const float* p10, const float* p11, int n_img,
                                     int H, int W, int C, float* out, void* stream) {
  STP3_CHECK_ARG(out && n_img > 0 && H > 0 && W > 0 && C > 0, "stp3_phase_interleave: bad argument");
  Phases ph{{p00, p01, p10, p11}};
  const long long total = (long long)n_img * H * W * C;
  phase_interleave_kernel<<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(ph, H, W, C, total, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_sigmoid_bwd(const float* g, const float* s, long long n, float* dz, void* stream) {
  STP3_CHECK_ARG(g && s && dz && n > 0, "stp3_sigmoid_bwd: bad argument");
  sigmoid_bwd_kernel<<<blocks_for(n), 256, 0, (cudaStream_t)stream>>>(g, s, n, dz);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_temporal_pair_mean(const float* m, int B, int T, int C, int adjoint, float* out, void* stream) {
  STP3_CHECK_ARG(m && out && B > 0 && T > 0 && C > 0, "stp3_temporal_pair_mean: bad argument");
  STP3_CHECK_ARG(m != out, "stp3_temporal_pair_mean: out must not alias m");
  const long long total = (long long)B * (adjoint ? T : T + 1) * C;
  temporal_pair_mean_kernel<<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(m, T, C, total, adjoint != 0, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
