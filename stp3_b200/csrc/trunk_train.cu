// Train mode of the EfficientNet trunk (efficientnet-pytorch 0.7.0 MBConv blocks, include/stp3_b200.h "EfficientNet
// trunk, train mode"): the raw stem and depthwise convolutions and their gradients, the BatchNorm apply / gradient pass
// with swish, squeeze-excite gate and drop-connect terms, and the squeeze-excite backward.  The 1x1 expand and
// projection convolutions, their gradients, the batch statistics and the BatchNorm backward are the train-mode kernels
// of train_kernels.cu / conv_igemm.cu.
//
// Tensors are fp32 channels-last, C channels per pixel row.  Every reduction writes per-block partials that a second
// kernel adds in a fixed order: no atomics, so every result is bitwise repeatable.
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace stp3 {
namespace {

constexpr int kTrThreads = 256;
constexpr int kTrStemMaxCout = 64;
constexpr int kTrMaxParts = 256;

inline unsigned tr_blocks(long long n) { return (unsigned)((n + kTrThreads - 1) / kTrThreads); }
inline int tr_parts(long long rows, long long rows_per_part) {
  const long long p = (rows + rows_per_part - 1) / rows_per_part;
  return (int)(p < 1 ? 1 : p > kTrMaxParts ? kTrMaxParts : p);
}

__device__ __forceinline__ float tr_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

// out[j] = sum over parts b = 0, 1, ... of part[b * n + j], in part order
__global__ void ordered_sum_kernel(const double* __restrict__ part, int n_part, long long n, float* __restrict__ out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double s = 0.0;
  for (int b = 0; b < n_part; ++b) s += part[(long long)b * n + j];
  out[j] = (float)s;
}

// ---------------------------------------------------------------- stem
// y (n_img, Ho, Wo, cout) = 3x3 stride-2 conv of the NCHW images, no bias, no activation; one thread per output element
__global__ void __launch_bounds__(kTrThreads)
stem_raw_kernel(const float* __restrict__ x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                const float* __restrict__ w, int cout, float* __restrict__ y) {
  __shared__ float sw[kTrStemMaxCout * 27];
  for (int i = threadIdx.x; i < cout * 27; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n_img * Ho * Wo * cout) return;
  const int c = (int)(idx % cout);
  const long long pix = idx / cout;
  const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), img = (int)(pix / ((long long)Wo * Ho));
  float a = 0.f;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int iy = oy * 2 - pad_t + ky, ix = ox * 2 - pad_l + kx;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W)
          a = fmaf(sw[c * 27 + (ci * 3 + ky) * 3 + kx], x[(((size_t)img * 3 + ci) * H + iy) * W + ix], a);
      }
  y[idx] = a;
}

// dW partials: CTA b owns a contiguous range of output pixels and walks it in chunks of kStemChunk pixels staged in
// shared memory (g rows and the 27 input taps of each pixel); thread j accumulates outputs j, j + 256, ... (cout * 27 of
// them) in fp64 over its CTA's pixels in pixel order -> part[b][cout * 27]
constexpr int kStemChunk = 32, kStemAccs = (kTrStemMaxCout * 27 + kTrThreads - 1) / kTrThreads;
__global__ void __launch_bounds__(kTrThreads)
stem_wgrad_partial_kernel(const float* __restrict__ x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                          const float* __restrict__ g, int cout, double* __restrict__ part) {
  __shared__ float sg[kStemChunk][kTrStemMaxCout];
  __shared__ float sx[kStemChunk][28];
  const long long n_pix = (long long)n_img * Ho * Wo;
  const long long per = (n_pix + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * per, p1 = p0 + per < n_pix ? p0 + per : n_pix;
  const int n_out = cout * 27;
  double acc[kStemAccs];
#pragma unroll
  for (int r = 0; r < kStemAccs; ++r) acc[r] = 0.0;
  for (long long q0 = p0; q0 < p1; q0 += kStemChunk) {
    __syncthreads();
    for (int i = threadIdx.x; i < kStemChunk * cout; i += blockDim.x) {
      const int pi = i / cout, c = i % cout;
      const long long p = q0 + pi;
      sg[pi][c] = p < p1 ? g[p * cout + c] : 0.f;
    }
    for (int i = threadIdx.x; i < kStemChunk * 27; i += blockDim.x) {
      const int pi = i / 27, t = i % 27;
      const long long p = q0 + pi;
      float v = 0.f;
      if (p < p1) {
        const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho), img = (int)(p / ((long long)Wo * Ho));
        const int ci = t / 9, iy = oy * 2 - pad_t + (t / 3) % 3, ix = ox * 2 - pad_l + t % 3;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)img * 3 + ci) * H + iy) * W + ix];
      }
      sx[pi][t] = v;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kStemAccs; ++r) {
      const int j = threadIdx.x + r * kTrThreads;
      if (j < n_out) {
        const int c = j / 27, t = j % 27;
        double s = acc[r];
        for (int pi = 0; pi < kStemChunk; ++pi) s = fma((double)sg[pi][c], (double)sx[pi][t], s);
        acc[r] = s;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kStemAccs; ++r) {
    const int j = threadIdx.x + r * kTrThreads;
    if (j < n_out) part[(size_t)blockIdx.x * n_out + j] = acc[r];
  }
}

// ---------------------------------------------------------------- depthwise
// y[img][oy][ox][c] = sum_{ky, kx} w[ky*k + kx][c] * x[img][oy*s - pad_t + ky][ox*s - pad_l + kx][c] (zero outside)
__global__ void __launch_bounds__(kTrThreads)
dw_raw_kernel(const stp3_dw_desc d, const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)d.n_img * d.Ho * d.Wo * d.C) return;
  const int c = (int)(idx % d.C);
  const long long pix = idx / d.C;
  const int ox = (int)(pix % d.Wo), oy = (int)((pix / d.Wo) % d.Ho), img = (int)(pix / ((long long)d.Wo * d.Ho));
  float a = 0.f;
  for (int ky = 0; ky < d.k; ++ky) {
    const int iy = oy * d.stride - d.pad_t + ky;
    if (iy < 0 || iy >= d.H) continue;
    for (int kx = 0; kx < d.k; ++kx) {
      const int ix = ox * d.stride - d.pad_l + kx;
      if (ix < 0 || ix >= d.W) continue;
      a = fmaf(w[(ky * d.k + kx) * d.C + c], x[(((size_t)img * d.H + iy) * d.W + ix) * d.in_cstride + c], a);
    }
  }
  y[pix * d.out_cstride + c] = a;
}

// The exact adjoint of dw_raw_kernel: input pixel iy receives tap ky from output row oy = (iy + pad_t - ky) / s when
// that division is exact and 0 <= oy < Ho (so rows the forward never read, past the bottom / right, get zero)
__global__ void __launch_bounds__(kTrThreads)
dw_dgrad_kernel(const stp3_dw_desc d, const float* __restrict__ g, const float* __restrict__ w, float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)d.n_img * d.H * d.W * d.C) return;
  const int c = (int)(idx % d.C);
  const long long pix = idx / d.C;
  const int ix = (int)(pix % d.W), iy = (int)((pix / d.W) % d.H), img = (int)(pix / ((long long)d.W * d.H));
  float a = 0.f;
  for (int ky = 0; ky < d.k; ++ky) {
    const int ty = iy + d.pad_t - ky;
    if (ty < 0 || ty % d.stride) continue;
    const int oy = ty / d.stride;
    if (oy >= d.Ho) continue;
    for (int kx = 0; kx < d.k; ++kx) {
      const int tx = ix + d.pad_l - kx;
      if (tx < 0 || tx % d.stride) continue;
      const int ox = tx / d.stride;
      if (ox >= d.Wo) continue;
      a = fmaf(w[(ky * d.k + kx) * d.C + c], g[(((size_t)img * d.Ho + oy) * d.Wo + ox) * d.out_cstride + c], a);
    }
  }
  dx[pix * d.in_cstride + c] = a;
}

// dW partials: grid (channel tiles of 32, parts), block (32, 8); thread (c, r) accumulates the K*K taps in fp64 over
// output pixels p0 + r, p0 + r + 8, ... of its part; the 8 rows are added in row order -> part[b][tap][C]
template <int K>
__global__ void __launch_bounds__(256)
dw_wgrad_partial_kernel(const stp3_dw_desc d, const float* __restrict__ x, const float* __restrict__ g,
                        double* __restrict__ part) {
  __shared__ double red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long n_pix = (long long)d.n_img * d.Ho * d.Wo;
  const long long per = (n_pix + gridDim.y - 1) / gridDim.y;
  const long long p0 = (long long)blockIdx.y * per, p1 = p0 + per < n_pix ? p0 + per : n_pix;
  double acc[K * K];
#pragma unroll
  for (int t = 0; t < K * K; ++t) acc[t] = 0.0;
  if (c < d.C) {
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const int ox = (int)(p % d.Wo), oy = (int)((p / d.Wo) % d.Ho), img = (int)(p / ((long long)d.Wo * d.Ho));
      const double gv = g[p * d.out_cstride + c];
#pragma unroll
      for (int ky = 0; ky < K; ++ky) {
        const int iy = oy * d.stride - d.pad_t + ky;
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const int ix = ox * d.stride - d.pad_l + kx;
          if (iy >= 0 && iy < d.H && ix >= 0 && ix < d.W)
            acc[ky * K + kx] = fma(gv, (double)x[(((size_t)img * d.H + iy) * d.W + ix) * d.in_cstride + c],
                                   acc[ky * K + kx]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < K * K; ++t) {
    red[threadIdx.y][threadIdx.x] = acc[t];
    __syncthreads();
    if (threadIdx.y == 0 && c < d.C) {
      double s = 0.0;
      for (int r = 0; r < 8; ++r) s += red[r][threadIdx.x];
      part[((size_t)blockIdx.y * K * K + t) * d.C + c] = s;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- BatchNorm apply / gradient with the trunk's terms
// y = act(z) * mul[img][c] * scale[img] + res, z = (x - mean) * invstd * gamma + beta (x itself when mean is NULL),
// act = swish or the identity; img = pixel / img_pix.  One thread per element of n_cols = max(C, hl_cs) columns:
// columns [C, hl_cs) of the planes are written as zeros.
__global__ void __launch_bounds__(kTrThreads)
trunk_bn_act_kernel(const float* __restrict__ x, long long n_pix, int C, long long img_pix, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                    int swish, const float* __restrict__ mul, const float* __restrict__ scale,
                    const float* __restrict__ res, float* __restrict__ y, __nv_bfloat16* __restrict__ yh,
                    __nv_bfloat16* __restrict__ yl, int hl_cs, int n_cols) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * n_cols) return;
  const int c = (int)(i % n_cols);
  const long long p = i / n_cols;
  float v = 0.f;
  if (c < C) {
    const long long img = p / img_pix;
    v = x[p * C + c];
    if (mean) v = (v - mean[c]) * invstd[c] * gamma[c] + beta[c];
    if (swish) v = v * tr_sigmoid(v);
    if (mul) v *= mul[img * C + c];
    if (scale) v *= scale[img];
    if (res) v += res[p * C + c];
    if (y) y[p * C + c] = v;
  }
  if (yh && c < hl_cs) ptx::split_hilo(v, yh[p * hl_cs + c], yl[p * hl_cs + c]);
}

// out = (g * mul[img][c] + add[img][c]) * act'(z) * scale[img], z recomputed from x and the statistics as above
// (swish'(z) = s (1 + z (1 - s)), s = sigmoid(z)); the dL/dz that the BatchNorm backward reduces
__global__ void __launch_bounds__(kTrThreads)
trunk_bn_act_bwd_kernel(const float* __restrict__ g, const float* __restrict__ x, long long n_pix, int C,
                        long long img_pix, const float* __restrict__ mean, const float* __restrict__ invstd,
                        const float* __restrict__ gamma, const float* __restrict__ beta, int swish,
                        const float* __restrict__ mul, const float* __restrict__ add, const float* __restrict__ scale,
                        float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * C) return;
  const int c = (int)(i % C);
  const long long p = i / C;
  const long long img = p / img_pix;
  float gv = g[i];
  if (mul) gv *= mul[img * C + c];
  if (add) gv += add[img * C + c];
  if (swish) {
    const float z = (x[i] - mean[c]) * invstd[c] * gamma[c] + beta[c];
    const float s = tr_sigmoid(z);
    gv *= s * (1.f + z * (1.f - s));
  }
  if (scale) gv *= scale[img];
  out[i] = gv;
}

// ---------------------------------------------------------------- squeeze-excite backward
// Per-image dot products over pixels: grid (channel tiles of 32, parts, images), block (32, 8), fp64 -> part[img][b][C]
__global__ void __launch_bounds__(256)
image_channel_dot_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, long long hw, int C,
                                 double* __restrict__ part) {
  __shared__ double red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long per = (hw + gridDim.y - 1) / gridDim.y;
  const long long p0 = (long long)blockIdx.y * per, p1 = p0 + per < hw ? p0 + per : hw;
  const size_t base = (size_t)blockIdx.z * hw * C;
  double s = 0.0;
  if (c < C)
    for (long long p = p0 + threadIdx.y; p < p1; p += 8)
      s = fma((double)a[base + p * C + c], (double)b[base + p * C + c], s);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t = 0.0;
    for (int r = 0; r < 8; ++r) t += red[r][threadIdx.x];
    part[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * C + c] = t;
  }
}

__global__ void image_channel_dot_finalize_kernel(const double* __restrict__ part, int n_part, int C,
                                                  float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const size_t img = blockIdx.y;
  double s = 0.0;
  for (int b = 0; b < n_part; ++b) s += part[(img * n_part + b) * C + c];
  out[img * C + c] = (float)s;
}

// One CTA per image: m = sums * inv_hw, r = w_r m + b_r (stp3_se_gate's order), de = dgate * gate * (1 - gate),
// d swish(r) = w_e^T de, dr = d swish(r) * swish'(r), dmean = (w_r^T dr) * inv_hw
__global__ void __launch_bounds__(256)
se_bwd_kernel(const float* __restrict__ dgate, const float* __restrict__ gate, const float* __restrict__ sums, int C,
              float inv_hw, const float* __restrict__ w_r, const float* __restrict__ b_r, int R,
              const float* __restrict__ w_e, float* __restrict__ de, float* __restrict__ sr, float* __restrict__ dr,
              float* __restrict__ dmean) {
  extern __shared__ float sm[];
  float* m = sm;                // [C]
  float* e = m + C;             // [C]
  float* d = e + C;             // [R]
  const size_t img = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    m[c] = sums[img * C + c] * inv_hw;
    const float gt = gate[img * C + c];
    e[c] = dgate[img * C + c] * (gt * (1.f - gt));
    de[img * C + c] = e[c];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = warp; j < R; j += nw) {
    float a = 0.f, b = 0.f;
    for (int c = lane; c < C; c += 32) {
      a = fmaf(w_r[(size_t)j * C + c], m[c], a);
      b = fmaf(w_e[(size_t)c * R + j], e[c], b);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, off);
      b += __shfl_xor_sync(0xffffffffu, b, off);
    }
    if (lane == 0) {
      const float r = a + b_r[j], s = tr_sigmoid(r);
      sr[img * R + j] = r * s;
      d[j] = b * (s * (1.f + r * (1.f - s)));
      dr[img * R + j] = d[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < R; ++j) a = fmaf(w_r[(size_t)j * C + c], d[j], a);
    dmean[img * C + c] = a * inv_hw;
  }
}

}  // namespace
}  // namespace stp3

using namespace stp3;

static int tr_check_dw(const stp3_dw_desc* d, const char* fn) {
  STP3_CHECK_ARG(d != nullptr, "%s: null descriptor", fn);
  STP3_CHECK_ARG(d->n_img > 0 && d->H > 0 && d->W > 0 && d->Ho > 0 && d->Wo > 0 && d->C > 0,
                 "%s: non-positive dimension", fn);
  STP3_CHECK_ARG(d->k == 3 || d->k == 5, "%s: k must be 3 or 5", fn);
  STP3_CHECK_ARG(d->stride == 1 || d->stride == 2, "%s: stride must be 1 or 2", fn);
  STP3_CHECK_ARG(d->pad_t >= 0 && d->pad_l >= 0 && d->pad_t < d->k && d->pad_l < d->k, "%s: pad out of range", fn);
  STP3_CHECK_ARG(d->in_cstride >= d->C && d->out_cstride >= d->C, "%s: a row stride is smaller than C", fn);
  return STP3_OK;
}

static int tr_check_stem(int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, int cout, const char* fn) {
  STP3_CHECK_ARG(n_img > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "%s: non-positive dimension", fn);
  STP3_CHECK_ARG(cout > 0 && cout <= kTrStemMaxCout, "%s: cout must be in [1, 64]", fn);
  STP3_CHECK_ARG(pad_t >= 0 && pad_l >= 0 && pad_t < 3 && pad_l < 3, "%s: pad out of range", fn);
  return STP3_OK;
}

extern "C" int stp3_effnet_stem_raw(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                                    const float* w, int cout, float* y, void* stream) {
  STP3_CHECK_ARG(x && w && y, "stp3_effnet_stem_raw: null pointer argument");
  const int rc = tr_check_stem(n_img, H, W, Ho, Wo, pad_t, pad_l, cout, "stp3_effnet_stem_raw");
  if (rc != STP3_OK) return rc;
  stem_raw_kernel<<<tr_blocks((long long)n_img * Ho * Wo * cout), kTrThreads, 0, (cudaStream_t)stream>>>(
      x, n_img, H, W, Ho, Wo, pad_t, pad_l, w, cout, y);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

static int stem_wgrad_parts(int n_img, int Ho, int Wo) { return tr_parts((long long)n_img * Ho * Wo, 1024); }

extern "C" size_t stp3_effnet_stem_wgrad_scratch_bytes(int n_img, int Ho, int Wo, int cout) {
  if (n_img <= 0 || Ho <= 0 || Wo <= 0 || cout <= 0) return 0;
  return (size_t)stem_wgrad_parts(n_img, Ho, Wo) * cout * 27 * sizeof(double);
}

extern "C" int stp3_effnet_stem_wgrad(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                                      const float* g, int cout, float* dw, void* scratch, size_t scratch_bytes,
                                      void* stream) {
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_effnet_stem_wgrad: null pointer argument");
  const int rc = tr_check_stem(n_img, H, W, Ho, Wo, pad_t, pad_l, cout, "stp3_effnet_stem_wgrad");
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(scratch_bytes >= stp3_effnet_stem_wgrad_scratch_bytes(n_img, Ho, Wo, cout),
                 "stp3_effnet_stem_wgrad: scratch smaller than stp3_effnet_stem_wgrad_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = stem_wgrad_parts(n_img, Ho, Wo);
  double* part = static_cast<double*>(scratch);
  stem_wgrad_partial_kernel<<<parts, kTrThreads, 0, st>>>(x, n_img, H, W, Ho, Wo, pad_t, pad_l, g, cout, part);
  STP3_CUDA_OK(cudaGetLastError());
  ordered_sum_kernel<<<tr_blocks(cout * 27), kTrThreads, 0, st>>>(part, parts, (long long)cout * 27, dw);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_dw_fwd_raw(const stp3_dw_desc* d, const float* x, const float* w, float* y, void* stream) {
  const int rc = tr_check_dw(d, "stp3_dw_fwd_raw");
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(x && w && y, "stp3_dw_fwd_raw: null pointer argument");
  dw_raw_kernel<<<tr_blocks((long long)d->n_img * d->Ho * d->Wo * d->C), kTrThreads, 0, (cudaStream_t)stream>>>(*d, x, w, y);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_dw_dgrad(const stp3_dw_desc* d, const float* g, const float* w, float* dx, void* stream) {
  const int rc = tr_check_dw(d, "stp3_dw_dgrad");
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(g && w && dx, "stp3_dw_dgrad: null pointer argument");
  dw_dgrad_kernel<<<tr_blocks((long long)d->n_img * d->H * d->W * d->C), kTrThreads, 0, (cudaStream_t)stream>>>(*d, g, w, dx);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

static int dw_wgrad_parts(const stp3_dw_desc* d) { return tr_parts((long long)d->n_img * d->Ho * d->Wo, 512); }

extern "C" size_t stp3_dw_wgrad_scratch_bytes(const stp3_dw_desc* d) {
  if (!d || d->n_img <= 0 || d->Ho <= 0 || d->Wo <= 0 || d->C <= 0 || d->k <= 0) return 0;
  return (size_t)dw_wgrad_parts(d) * d->k * d->k * d->C * sizeof(double);
}

extern "C" int stp3_dw_wgrad(const stp3_dw_desc* d, const float* x, const float* g, float* dw, void* scratch,
                             size_t scratch_bytes, void* stream) {
  const int rc = tr_check_dw(d, "stp3_dw_wgrad");
  if (rc != STP3_OK) return rc;
  STP3_CHECK_ARG(x && g && dw && scratch, "stp3_dw_wgrad: null pointer argument");
  STP3_CHECK_ARG(scratch_bytes >= stp3_dw_wgrad_scratch_bytes(d),
                 "stp3_dw_wgrad: scratch smaller than stp3_dw_wgrad_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = dw_wgrad_parts(d);
  double* part = static_cast<double*>(scratch);
  const dim3 grid(ceil_div(d->C, 32), parts), block(32, 8);
  if (d->k == 3)
    dw_wgrad_partial_kernel<3><<<grid, block, 0, st>>>(*d, x, g, part);
  else
    dw_wgrad_partial_kernel<5><<<grid, block, 0, st>>>(*d, x, g, part);
  STP3_CUDA_OK(cudaGetLastError());
  const long long n = (long long)d->k * d->k * d->C;
  ordered_sum_kernel<<<tr_blocks(n), kTrThreads, 0, st>>>(part, parts, n, dw);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_trunk_bn_act(const float* x, long long n_pix, int C, long long img_pix, const float* mean,
                                 const float* invstd, const float* gamma, const float* beta, int swish,
                                 const float* mul, const float* scale, const float* res, float* y, void* y_hi,
                                 void* y_lo, int hl_cstride, void* stream) {
  STP3_CHECK_ARG(x && (y || y_hi) && n_pix > 0 && C > 0 && img_pix > 0 && n_pix % img_pix == 0,
                 "stp3_trunk_bn_act: bad argument");
  STP3_CHECK_ARG(!mean || (invstd && gamma && beta), "stp3_trunk_bn_act: mean needs invstd, gamma and beta");
  STP3_CHECK_ARG((y_hi == nullptr) == (y_lo == nullptr), "stp3_trunk_bn_act: give both bf16 planes or neither");
  STP3_CHECK_ARG(!y_hi || hl_cstride >= C, "stp3_trunk_bn_act: plane row stride smaller than C");
  const int n_cols = y_hi ? hl_cstride : C;
  trunk_bn_act_kernel<<<tr_blocks(n_pix * n_cols), kTrThreads, 0, (cudaStream_t)stream>>>(
      x, n_pix, C, img_pix, mean, invstd, gamma, beta, swish, mul, scale, res, y, (__nv_bfloat16*)y_hi,
      (__nv_bfloat16*)y_lo, y_hi ? hl_cstride : 0, n_cols);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_trunk_bn_act_bwd(const float* g, const float* x, long long n_pix, int C, long long img_pix,
                                     const float* mean, const float* invstd, const float* gamma, const float* beta,
                                     int swish, const float* mul, const float* add, const float* scale, float* out,
                                     void* stream) {
  STP3_CHECK_ARG(g && out && n_pix > 0 && C > 0 && img_pix > 0 && n_pix % img_pix == 0,
                 "stp3_trunk_bn_act_bwd: bad argument");
  STP3_CHECK_ARG(!swish || (x && mean && invstd && gamma && beta),
                 "stp3_trunk_bn_act_bwd: swish needs x, mean, invstd, gamma and beta");
  trunk_bn_act_bwd_kernel<<<tr_blocks(n_pix * C), kTrThreads, 0, (cudaStream_t)stream>>>(
      g, x, n_pix, C, img_pix, mean, invstd, gamma, beta, swish, mul, add, scale, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

static int dot_parts(long long hw) { return tr_parts(hw, 256); }

extern "C" size_t stp3_image_channel_dot_scratch_bytes(int n_img, long long hw, int C) {
  if (n_img <= 0 || hw <= 0 || C <= 0) return 0;
  return (size_t)n_img * dot_parts(hw) * C * sizeof(double);
}

extern "C" int stp3_image_channel_dot(const float* a, const float* b, int n_img, long long hw, int C, float* out,
                                      void* scratch, size_t scratch_bytes, void* stream) {
  STP3_CHECK_ARG(a && b && out && scratch && n_img > 0 && hw > 0 && C > 0, "stp3_image_channel_dot: bad argument");
  STP3_CHECK_ARG(n_img <= 65535, "stp3_image_channel_dot: more than 65535 images");
  STP3_CHECK_ARG(scratch_bytes >= stp3_image_channel_dot_scratch_bytes(n_img, hw, C),
                 "stp3_image_channel_dot: scratch smaller than stp3_image_channel_dot_scratch_bytes()");
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = dot_parts(hw);
  double* part = static_cast<double*>(scratch);
  image_channel_dot_partial_kernel<<<dim3(ceil_div(C, 32), parts, n_img), dim3(32, 8), 0, st>>>(a, b, hw, C, part);
  STP3_CUDA_OK(cudaGetLastError());
  image_channel_dot_finalize_kernel<<<dim3(ceil_div(C, 128), n_img), 128, 0, st>>>(part, parts, C, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_se_bwd(const float* dgate, const float* gate, const float* sums, int n_img, int C, float inv_hw,
                           const float* w_r, const float* b_r, int R, const float* w_e, float* de, float* sr, float* dr,
                           float* dmean, void* stream) {
  STP3_CHECK_ARG(dgate && gate && sums && w_r && b_r && w_e && de && sr && dr && dmean, "stp3_se_bwd: null pointer argument");
  STP3_CHECK_ARG(n_img > 0 && C > 0 && R > 0 && C <= 4096 && R <= 1024, "stp3_se_bwd: bad dimensions");
  se_bwd_kernel<<<n_img, 256, (size_t)(2 * C + R) * sizeof(float), (cudaStream_t)stream>>>(
      dgate, gate, sums, C, inv_hw, w_r, b_r, R, w_e, de, sr, dr, dmean);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
