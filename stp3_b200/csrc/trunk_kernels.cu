// The memory-bound layers of the EfficientNet trunk (efficientnet-pytorch 0.7.0 MBConv blocks; the 1x1 expand and project
// convolutions run on stp3_conv_fwd): the stem convolution, the depthwise convolution with the squeeze-excite spatial
// sums, and the squeeze-excite gate folded into per-image projection weights.
//
// Static "same" padding: the pads are computed by the caller for the model's nominal image size (0.7.0 builds
// Conv2dStaticSamePadding with image_size); the kernels take the top / left pad and the output size, and every input
// coordinate outside the image reads as zero (which is the bottom / right pad).
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace stp3 {

__device__ __forceinline__ float swish(float v) { return v / (1.f + __expf(-v)); }

// ---------------------------------------------------------------- stem
// fp32 NCHW (n_img, 3, H, W) -> 3x3 stride-2 conv + folded BN + swish -> hi/lo (n_img, Ho, Wo, cstride), channels >= cout
// zero.  A thread owns one output pixel and 16 channels; the weights sit in shared memory.
constexpr int kStemMaxCout = 64;
__global__ void __launch_bounds__(256)
stem_kernel(const float* __restrict__ x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
            const float* __restrict__ w, const float* __restrict__ bias, int cout, int cstride,
            __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
  __shared__ float sw[kStemMaxCout * 27];
  __shared__ float sb[kStemMaxCout];
  ptx::griddep_wait();
  for (int i = threadIdx.x; i < cout * 27; i += blockDim.x) sw[i] = w[i];
  for (int i = threadIdx.x; i < cout; i += blockDim.x) sb[i] = bias[i];
  __syncthreads();
  const int n_cg = cstride / 16;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_pix = (long long)n_img * Ho * Wo;
  if (idx >= n_pix * n_cg) return;
  const int cg = (int)(idx % n_cg);
  const long long pix = idx / n_cg;
  const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), img = (int)(pix / ((long long)Wo * Ho));
  float in[27];
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int iy = oy * 2 - pad_t + ky, ix = ox * 2 - pad_l + kx;
        in[(ci * 3 + ky) * 3 + kx] =
            (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[(((size_t)img * 3 + ci) * H + iy) * W + ix] : 0.f;
      }
  uint32_t hw[8], lw[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = cg * 16 + 2 * j + e;
      float a = 0.f;
      if (c < cout) {
        a = sb[c];
#pragma unroll
        for (int t = 0; t < 27; ++t) a = fmaf(sw[c * 27 + t], in[t], a);
        a = swish(a);
      }
      v[e] = a;
    }
    ptx::split_hilo(v[0], v[1], hw[j], lw[j]);
  }
  const size_t off = (size_t)pix * cstride + cg * 16;
  uint4* ph = reinterpret_cast<uint4*>(y_hi + off);
  uint4* pl = reinterpret_cast<uint4*>(y_lo + off);
  ph[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]); ph[1] = make_uint4(hw[4], hw[5], hw[6], hw[7]);
  pl[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]); pl[1] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
}

// ---------------------------------------------------------------- depthwise
// CTA = one 8 x 16 output tile x 64 channels of one image; thread = 8 channels (one 16-byte vector per plane) of four
// pixels of the tile.  A warp covers 4 neighbouring pixels x 64 channels, so every load is 4 x 128 contiguous bytes per
// plane; the k*k taps of neighbouring pixels overlap and are served from L1, so HBM sees each input byte about once.
// Squeeze-excite sums: each CTA writes one partial row (its tile's sums, fixed-order reduction over its pixel slots) to
// scratch; dw_sum_reduce_kernel adds the rows of an image in tile order.  No atomics: bitwise repeatable.
constexpr int kDwTileH = 8, kDwTileW = 16, kDwThreads = 256, kDwMaxK = 5;
__global__ void __launch_bounds__(kDwThreads)
dw_kernel(const stp3_dw_desc d, const __nv_bfloat16* __restrict__ x_hi, const __nv_bfloat16* __restrict__ x_lo,
          const float* __restrict__ w, const float* __restrict__ bias, __nv_bfloat16* __restrict__ y_hi,
          __nv_bfloat16* __restrict__ y_lo, float* __restrict__ part, int tiles_x, int n_tiles) {
  __shared__ float sw[kDwMaxK * kDwMaxK * 64];
  __shared__ float sb[64];
  __shared__ float red[32][65];
  ptx::griddep_wait();
  const int tile = blockIdx.x, cblk = blockIdx.y, img = blockIdx.z;
  const int cbase = cblk * 64;
  const int kk = d.k * d.k;
  for (int i = threadIdx.x; i < kk * 64; i += kDwThreads) {
    const int t = i / 64, c = cbase + i % 64;
    sw[i] = c < d.C ? w[(size_t)t * d.C + c] : 0.f;
  }
  for (int i = threadIdx.x; i < 64; i += kDwThreads) sb[i] = cbase + i < d.C ? bias[cbase + i] : 0.f;
  __syncthreads();
  const int cv = threadIdx.x & 7, slot = threadIdx.x >> 3;
  const int c0 = cbase + cv * 8;
  const bool c_ok = c0 < d.C;
  const int oy0 = (tile / tiles_x) * kDwTileH, ox0 = (tile % tiles_x) * kDwTileW;
  float sum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sum[i] = 0.f;
#pragma unroll 1
  for (int j = 0; j < 4; ++j) {
    const int pi = slot + 32 * j;
    const int oy = oy0 + pi / kDwTileW, ox = ox0 + pi % kDwTileW;
    if (!c_ok || oy >= d.Ho || ox >= d.Wo) continue;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int ky = 0; ky < d.k; ++ky) {
      const int iy = oy * d.stride - d.pad_t + ky;
      if (iy < 0 || iy >= d.H) continue;
      for (int kx = 0; kx < d.k; ++kx) {
        const int ix = ox * d.stride - d.pad_l + kx;
        if (ix < 0 || ix >= d.W) continue;
        const size_t off = (((size_t)img * d.H + iy) * d.W + ix) * d.in_cstride + c0;
        const uint4 h4 = __ldg(reinterpret_cast<const uint4*>(x_hi + off));
        const uint4 l4 = __ldg(reinterpret_cast<const uint4*>(x_lo + off));
        const uint32_t hh[4] = {h4.x, h4.y, h4.z, h4.w}, ll[4] = {l4.x, l4.y, l4.z, l4.w};
        const float* wt = sw + (ky * d.k + kx) * 64 + cv * 8;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 v = ptx::join_hilo(hh[e], ll[e]);
          acc[2 * e] = fmaf(wt[2 * e], v.x, acc[2 * e]);
          acc[2 * e + 1] = fmaf(wt[2 * e + 1], v.y, acc[2 * e + 1]);
        }
      }
    }
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a0 = swish(acc[2 * e] + sb[cv * 8 + 2 * e]), a1 = swish(acc[2 * e + 1] + sb[cv * 8 + 2 * e + 1]);
      sum[2 * e] += a0; sum[2 * e + 1] += a1;
      ptx::split_hilo(a0, a1, hw[e], lw[e]);
    }
    const size_t o = (((size_t)img * d.Ho + oy) * d.Wo + ox) * d.out_cstride + c0;
    *reinterpret_cast<uint4*>(y_hi + o) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(y_lo + o) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
  if (part == nullptr) return;
#pragma unroll
  for (int i = 0; i < 8; ++i) red[slot][cv * 8 + i] = sum[i];
  __syncthreads();
  if (threadIdx.x < 64 && cbase + threadIdx.x < d.C) {
    float s = 0.f;
    for (int k = 0; k < 32; ++k) s += red[k][threadIdx.x];
    part[((size_t)img * n_tiles + tile) * d.C + cbase + threadIdx.x] = s;
  }
}

// sums[img][c] = sum over the tiles of the image's partial rows, in tile order
__global__ void dw_sum_reduce_kernel(const float* __restrict__ part, int n_tiles, int C, float* __restrict__ sums) {
  ptx::griddep_wait();
  const int img = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int t = 0; t < n_tiles; ++t) s += part[((size_t)img * n_tiles + t) * C + c];
  sums[(size_t)img * C + c] = s;
}

// ---------------------------------------------------------------- squeeze-excite gate -> per-image projection weights
// Two launches.  se_gate_kernel: one CTA per image computes its gate once (2 * C * R MACs).  se_scale_kernel: grid
// (n_img, slices), each CTA writes its slice of W_proj . diag(gate) as bf16 hi/lo in the packed layout of stp3_conv_fwd.
// The weights of a projection are stored as column chunks of at most 128 rows (a chunk of <= 64 real columns has
// bn = 64): chunk j at element offset sum_{j' < j} kblocks * 2 * bn_j' * 64 of the image's block, [kb][plane][bn_j][64].
__host__ __device__ __forceinline__ int chunk_bn(int rem) { return rem > 64 ? 128 : 64; }

__global__ void __launch_bounds__(256)
se_gate_kernel(const float* __restrict__ sums, int sums_stride, int C, float inv_hw, const float* __restrict__ w_r,
               const float* __restrict__ b_r, int R, const float* __restrict__ w_e, const float* __restrict__ b_e,
               float* __restrict__ gate) {
  extern __shared__ float sm[];
  float* m = sm;                       // [C]
  float* r = m + C;                    // [R]
  ptx::griddep_wait();
  const int img = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) m[c] = sums[(size_t)img * sums_stride + c] * inv_hw;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = warp; j < R; j += nw) {
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(w_r[(size_t)j * C + c], m[c], a);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
    if (lane == 0) r[j] = swish(a + b_r[j]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = b_e[c];
    for (int j = 0; j < R; ++j) a = fmaf(w_e[(size_t)c * R + j], r[j], a);
    gate[(size_t)img * C + c] = 1.f / (1.f + expf(-a));
  }
}

__global__ void __launch_bounds__(256)
se_scale_kernel(const float* __restrict__ gate, int C, const float* __restrict__ w_p, int cout, int kblocks,
                long long img_stride, __nv_bfloat16* __restrict__ w_img) {
  extern __shared__ float g[];         // [kblocks * 64]
  ptx::griddep_wait();                 // the gate comes from the preceding kernel
  const int img = blockIdx.x;
  for (int c = threadIdx.x; c < kblocks * 64; c += blockDim.x) g[c] = c < C ? gate[(size_t)img * C + c] : 0.f;
  __syncthreads();
  // element pairs (hi, lo) of the image's block: q enumerates (chunk, kb, row, k) with k fastest
  __nv_bfloat16* dst = w_img + (size_t)img * img_stride;
  long long chunk_off = 0;
  for (int n0 = 0; n0 < cout; n0 += 128) {
    const int bn = chunk_bn(cout - n0);
    const long long n_q = (long long)kblocks * bn * 64;
    for (long long q = (long long)blockIdx.y * blockDim.x + threadIdx.x; q < n_q; q += (long long)gridDim.y * blockDim.x) {
      const int k = (int)(q % 64), row = (int)((q / 64) % bn), kb = (int)(q / (64 * (long long)bn));
      const int n = n0 + row, c = kb * 64 + k;
      const float v = (n < cout && c < C) ? w_p[(size_t)n * C + c] * g[c] : 0.f;
      __nv_bfloat16 h, l;
      ptx::split_hilo(v, h, l);
      const long long o = chunk_off + ((long long)(kb * 2) * bn + row) * 64 + k;
      dst[o] = h;
      dst[o + (long long)bn * 64] = l;
    }
    chunk_off += (long long)kblocks * 2 * bn * 64;
  }
}

}  // namespace stp3

using namespace stp3;

extern "C" int stp3_effnet_stem(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                                const float* w, const float* bias, int cout, int out_cstride, void* y_hi, void* y_lo,
                                void* stream_) {
  STP3_CHECK_ARG(x && w && bias && y_hi && y_lo, "stp3_effnet_stem: null pointer argument");
  STP3_CHECK_ARG(n_img > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "stp3_effnet_stem: non-positive dimension");
  STP3_CHECK_ARG(cout > 0 && cout <= kStemMaxCout && out_cstride % 64 == 0 && out_cstride >= cout,
                 "stp3_effnet_stem: cout must be <= 64 and out_cstride a multiple of 64 >= cout");
  STP3_CHECK_ARG(pad_t >= 0 && pad_l >= 0 && pad_t < 3 && pad_l < 3, "stp3_effnet_stem: pad out of range");
  STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(y_hi) | reinterpret_cast<uintptr_t>(y_lo)) % 16 == 0,
                 "stp3_effnet_stem: y_hi / y_lo must be 16-byte aligned");
  const long long n = (long long)n_img * Ho * Wo * (out_cstride / 16);
  STP3_CHECK_ARG((n + 255) / 256 <= 0x7fffffffll, "stp3_effnet_stem: more than 2^31 - 1 blocks of 256 threads");
  const unsigned grid = (unsigned)((n + 255) / 256);
  STP3_CUDA_OK(launch_pdl(kPdlAux, stem_kernel, dim3(grid), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream_), x,
                          n_img, H, W, Ho, Wo, pad_t, pad_l, w, bias, cout, out_cstride,
                          static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo)));
  return STP3_OK;
}

static int dw_tiles(const stp3_dw_desc* d, int* tiles_x) {
  *tiles_x = ceil_div(d->Wo, kDwTileW);
  return *tiles_x * ceil_div(d->Ho, kDwTileH);
}

extern "C" size_t stp3_dw_sums_scratch_bytes(const stp3_dw_desc* d) {
  if (!d || d->n_img <= 0 || d->Ho <= 0 || d->Wo <= 0 || d->C <= 0) return 0;
  int tx;
  return (size_t)d->n_img * dw_tiles(d, &tx) * d->C * sizeof(float);
}

extern "C" int stp3_dw_fwd(const stp3_dw_desc* d, const void* x_hi, const void* x_lo, const float* w, const float* bias,
                           void* y_hi, void* y_lo, float* sums, void* scratch, size_t scratch_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STP3_CHECK_ARG(d && x_hi && x_lo && w && bias && y_hi && y_lo, "stp3_dw_fwd: null pointer argument");
  STP3_CHECK_ARG(d->n_img > 0 && d->H > 0 && d->W > 0 && d->Ho > 0 && d->Wo > 0, "stp3_dw_fwd: non-positive dimension");
  STP3_CHECK_ARG(d->k == 3 || d->k == 5, "stp3_dw_fwd: k must be 3 or 5");
  STP3_CHECK_ARG(d->stride == 1 || d->stride == 2, "stp3_dw_fwd: stride must be 1 or 2");
  STP3_CHECK_ARG(d->pad_t >= 0 && d->pad_l >= 0 && d->pad_t < d->k && d->pad_l < d->k, "stp3_dw_fwd: pad out of range");
  STP3_CHECK_ARG(d->C > 0 && d->C % 8 == 0 && d->in_cstride % 64 == 0 && d->out_cstride % 64 == 0 &&
                 d->C <= d->in_cstride && d->C <= d->out_cstride,
                 "stp3_dw_fwd: C must be a multiple of 8 inside channel strides that are multiples of 64");
  STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(x_hi) | reinterpret_cast<uintptr_t>(x_lo) | reinterpret_cast<uintptr_t>(y_hi) |
                  reinterpret_cast<uintptr_t>(y_lo)) % 16 == 0, "stp3_dw_fwd: planes must be 16-byte aligned");
  int tiles_x;
  const int n_tiles = dw_tiles(d, &tiles_x);
  float* part = nullptr;
  if (sums) {
    STP3_CHECK_ARG(scratch && scratch_bytes >= stp3_dw_sums_scratch_bytes(d),
                   "stp3_dw_fwd: sums scratch missing or smaller than stp3_dw_sums_scratch_bytes()");
    part = static_cast<float*>(scratch);
  }
  STP3_CHECK_ARG(d->n_img < 65536, "stp3_dw_fwd: too many images");
  STP3_CUDA_OK(launch_pdl(kPdlAux, dw_kernel, dim3(n_tiles, ceil_div(d->C, 64), d->n_img), dim3(kDwThreads), 0, stream,
                          *d, static_cast<const __nv_bfloat16*>(x_hi), static_cast<const __nv_bfloat16*>(x_lo), w, bias,
                          static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo), part, tiles_x, n_tiles));
  if (sums)
    STP3_CUDA_OK(launch_pdl(kPdlAux, dw_sum_reduce_kernel, dim3(ceil_div(d->C, 128), d->n_img), dim3(128), 0, stream,
                            (const float*)part, n_tiles, d->C, sums));
  return STP3_OK;
}

extern "C" long long stp3_se_proj_weight_elems(int cin, int cout) {
  if (cin <= 0 || cout <= 0) return 0;
  const long long kblocks = (cin + 63) / 64;
  long long n = 0;
  for (int n0 = 0; n0 < cout; n0 += 128) n += kblocks * 2 * chunk_bn(cout - n0) * 64;
  return n;
}

extern "C" int stp3_se_gate(const float* sums, int sums_stride, int n_img, int C, float inv_hw, const float* w_r,
                            const float* b_r, int R, const float* w_e, const float* b_e, const float* w_proj, int cout,
                            float* gate, void* w_img, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STP3_CHECK_ARG(sums && w_r && b_r && w_e && b_e && w_proj && gate && w_img, "stp3_se_gate: null pointer argument");
  STP3_CHECK_ARG(n_img > 0 && C > 0 && R > 0 && cout > 0 && sums_stride >= C, "stp3_se_gate: bad dimensions");
  STP3_CHECK_ARG(C <= 4096 && R <= 1024, "stp3_se_gate: C <= 4096 and R <= 1024");
  const int kblocks = (C + 63) / 64;
  const long long stride = stp3_se_proj_weight_elems(C, cout);
  STP3_CUDA_OK(launch_pdl(kPdlAux, se_gate_kernel, dim3(n_img), dim3(256), (size_t)(C + R) * sizeof(float), stream, sums,
                          sums_stride, C, inv_hw, w_r, b_r, R, w_e, b_e, gate));
  const int slices = (int)((stride / 2 + 256 * 8 - 1) / (256 * 8));
  STP3_CUDA_OK(launch_pdl(kPdlAux, se_scale_kernel, dim3(n_img, slices > 0 ? slices : 1), dim3(256),
                          (size_t)kblocks * 64 * sizeof(float), stream, (const float*)gate, C, w_proj, cout, kblocks,
                          stride, static_cast<__nv_bfloat16*>(w_img)));
  return STP3_OK;
}
