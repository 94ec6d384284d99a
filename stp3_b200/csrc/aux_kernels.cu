// Memory-bound helpers around the tensor-core path: layout / precision-split conversions, spatial sums, the tiny
// dense layers of the spatially constant branches, and the bilinear x2 upsample + skip add of UpsamplingAdd.
// All activations are channels-last bf16 hi/lo planes (see conv_igemm.cu).
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace stp3 {

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& h, __nv_bfloat16& l) {
  h = __float2bfloat16_rn(x);
  l = __float2bfloat16_rn(x - __bfloat162float(h));
}
__device__ __forceinline__ float join_bf16(__nv_bfloat16 h, __nv_bfloat16 l) {
  return __bfloat162float(h) + __bfloat162float(l);
}

// fp32 (n_img, C, H*W) [NCHW] or (n_img, H*W, C) [NHWC] -> hi/lo (n_img, H*W, cp), zero padding channels.
// 32 pixels x 32 channels per block through shared memory so that both sides are coalesced.
__global__ void __launch_bounds__(256)
f32_to_hilo_kernel(const float* __restrict__ x, int channels_last, int C, int HW, int cp,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float tile[32][33];
  const int img = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;   // (32, 8)
  if (!channels_last) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + ty + 8 * k, px = p0 + tx;
      tile[ty + 8 * k][tx] = (c < C && px < HW) ? x[((size_t)img * C + c) * HW + px] : 0.f;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int px = p0 + ty + 8 * k, c = c0 + tx;
      tile[tx][ty + 8 * k] = (c < C && px < HW) ? x[((size_t)img * HW + px) * C + c] : 0.f;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int px = p0 + ty + 8 * k, c = c0 + tx;
    if (px < HW && c < cp) {
      __nv_bfloat16 h, l;
      split_bf16(tile[tx][ty + 8 * k], h, l);
      hi[((size_t)img * HW + px) * cp + c] = h;
      lo[((size_t)img * HW + px) * cp + c] = l;
    }
  }
}

// hi/lo (n_img, H*W, cstride) channels [c_off, c_off+C) -> fp32 (n_img, C, H*W)
__global__ void __launch_bounds__(256)
hilo_to_f32_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int cstride, int c_off,
                   int C, int HW, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int img = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int px = p0 + ty + 8 * k, c = c0 + tx;
    float v = 0.f;
    if (px < HW && c < C) {
      const size_t i = ((size_t)img * HW + px) * cstride + c_off + c;
      v = join_bf16(hi[i], lo[i]);
    }
    tile[ty + 8 * k][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c0 + ty + 8 * k, px = p0 + tx;
    if (c < C && px < HW) out[((size_t)img * C + c) * HW + px] = tile[tx][ty + 8 * k];
  }
}

// sums[img][c] += sum over pixels of (hi+lo); grid (pixel chunks, n_img); block = cstride threads (<= 1024)
__global__ void spatial_sum_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                   int HW, int cstride, int px_per_block, float* __restrict__ sums) {
  const int img = blockIdx.y;
  const int c = threadIdx.x;
  const int p0 = blockIdx.x * px_per_block, p1 = min(HW, p0 + px_per_block);
  float acc = 0.f;
  for (int px = p0; px < p1; ++px) {
    const size_t i = ((size_t)img * HW + px) * cstride + c;
    acc += join_bf16(hi[i], lo[i]);
  }
  atomicAdd(sums + (size_t)img * cstride + c, acc);
}

// The spatially constant branches (PyramidSpatioTemporalPooling temporal.py:375-423, ASPPPooling convolutions.py:
// 227-239) collapse to a per-image vector:  m = mean over pixels (and, if temporal, over frames {t-1, t} that exist)
//   v = relu(W1 m + b1)   [R]        (1x1(x1) conv + folded BN + ReLU on a 1x1 map; bilinear resize of a constant)
//   out[img][co] (+)= sum_r W2[co][r] v[r]     (its slice of the consuming 1x1 convolution, folded BN scale inside)
// one block per image
__global__ void pool_bias_kernel(const float* __restrict__ sums, int sums_stride, int T, int C, float inv_hw,
                                 int temporal, const float* __restrict__ cvals, int n_const,
                                 const float* __restrict__ W1, const float* __restrict__ b1, int R,
                                 const float* __restrict__ W2, int CO, const float* __restrict__ bias,
                                 float* __restrict__ out, int co_stride, int accumulate) {
  ptx::griddep_launch_dependents();
  ptx::griddep_wait();                      // sums / constants come from the preceding kernels
  extern __shared__ float sm[];
  float* m = sm;          // [C]
  float* v = sm + C;      // [R]
  const int img = blockIdx.x;
  const int t = img % T;
  const int cs = C - n_const;       // channels [cs, C) are spatially constant: their per-frame mean is the value itself
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    auto frame_mean = [&](int i) {
      return c < cs ? sums[(size_t)i * sums_stride + c] * inv_hw : cvals[(size_t)i * n_const + (c - cs)];
    };
    float s = frame_mean(img);
    float cnt = 1.f;
    if (temporal && t > 0) { s += frame_mean(img - 1); cnt = 2.f; }
    m[c] = s / cnt;
  }
  __syncthreads();
  // one warp per output row, lanes stride over the inputs; four rows in flight per warp so that their (cold, L2 / HBM)
  // weight loads overlap -- the kernel sits on the critical path between two convolutions and is pure latency
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int r0 = warp * 4; r0 < R; r0 += nwarps * 4) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = lane; c < C; c += 32) {
      const float mc = m[c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (r0 + i < R) a[i] = fmaf(__ldg(W1 + (size_t)(r0 + i) * C + c), mc, a[i]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a[i] += __shfl_xor_sync(0xffffffffu, a[i], o);
      if (lane == 0 && r0 + i < R) v[r0 + i] = fmaxf(a[i] + b1[r0 + i], 0.f);
    }
  }
  __syncthreads();
  // blockIdx.y owns a slice of the output rows (every slice recomputes the small hidden vector v)
  const int co_per = (CO + gridDim.y - 1) / gridDim.y;
  const int co_begin = blockIdx.y * co_per, co_end = min(CO, co_begin + co_per);
  for (int co0 = co_begin + warp * 4; co0 < co_end; co0 += nwarps * 4) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = lane; r < R; r += 32) {
      const float vr = v[r];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (co0 + i < co_end) a[i] = fmaf(__ldg(W2 + (size_t)(co0 + i) * R + r), vr, a[i]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a[i] += __shfl_xor_sync(0xffffffffu, a[i], o);
      if (lane == 0 && co0 + i < co_end) {
        float* dst = out + (size_t)img * co_stride + co0 + i;
        *dst = (accumulate ? *dst : (bias ? bias[co0 + i] : 0.f)) + a[i];
      }
    }
  }
}

// y[n][co] (+)= sum_ci W[co][ci] x[n][ci]     (ego-motion channels folded into a per-image bias, stp3.py:145-152)
__global__ void small_linear_kernel(const float* __restrict__ x, const float* __restrict__ W, int ci, int co,
                                    const float* __restrict__ bias, float* __restrict__ y, int co_stride,
                                    int accumulate) {
  ptx::griddep_launch_dependents();
  ptx::griddep_wait();
  const int n = blockIdx.x;
  for (int o = threadIdx.x; o < co; o += blockDim.x) {
    float a = 0.f;
    for (int i = 0; i < ci; ++i) a = fmaf(W[(size_t)o * ci + i], x[(size_t)n * ci + i], a);
    float* dst = y + (size_t)n * co_stride + o;
    *dst = (accumulate ? *dst : (bias ? bias[o] : 0.f)) + a;
  }
}

// UpsamplingAdd tail (convolutions.py:204-215): y = bilinear_x2(x, align_corners=False) + skip.  The 1x1 conv + BN
// of the reference have already been applied at low resolution (they commute with the interpolation).
// one thread = one output pixel x 8 channels (16-byte vectors)
__global__ void __launch_bounds__(256)
upsample2x_add_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl, int h, int w, int xs,
                      const __nv_bfloat16* __restrict__ sh, const __nv_bfloat16* __restrict__ sl, int ss, int s_off,
                      __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int ys, int y_off, int C8,
                      size_t total) {
  ptx::griddep_launch_dependents();
  ptx::griddep_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = idx % C8;
  size_t r = idx / C8;
  const int W2 = 2 * w, H2 = 2 * h;
  const int ox = r % W2; r /= W2;
  const int oy = r % H2;
  const size_t img = r / H2;
  // PyTorch: src = (dst + 0.5) / 2 - 0.5, clamped at 0; weights (1 - frac, frac)
  const float fy = fmaxf((oy + 0.5f) * 0.5f - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * 0.5f - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float wy1 = fy - y0, wx1 = fx - x0, wy0 = 1.f - wy1, wx0 = 1.f - wx1;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const int ys_[2] = {y0, y1}, xs_[2] = {x0, x1};
  const float wys[2] = {wy0, wy1}, wxs[2] = {wx0, wx1};
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const size_t i = ((img * h + ys_[a]) * w + xs_[b]) * xs + g * 8;
      const uint4 hv = *reinterpret_cast<const uint4*>(xh + i), lv = *reinterpret_cast<const uint4*>(xl + i);
      const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, lw[4] = {lv.x, lv.y, lv.z, lv.w};
      // same evaluation order as ATen's upsample_bilinear2d: w_y * (w_x0 * v0 + w_x1 * v1) is reproduced to fp32
      // round-off by accumulating the four weighted corners
      const float wt = wys[a] * wxs[b];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        acc[2 * e] = fmaf(wt, __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16), acc[2 * e]);
        acc[2 * e + 1] = fmaf(wt, __uint_as_float(hw[e] & 0xFFFF0000u) + __uint_as_float(lw[e] & 0xFFFF0000u), acc[2 * e + 1]);
      }
    }
  const size_t opix = (img * H2 + oy) * W2 + ox;
  if (sh != nullptr) {
    const size_t i = opix * ss + s_off + g * 8;
    const uint4 hv = *reinterpret_cast<const uint4*>(sh + i), lv = *reinterpret_cast<const uint4*>(sl + i);
    const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, lw[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      acc[2 * e] += __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
      acc[2 * e + 1] += __uint_as_float(hw[e] & 0xFFFF0000u) + __uint_as_float(lw[e] & 0xFFFF0000u);
    }
  }
  uint32_t oh[4], ol[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    __nv_bfloat16 h0, l0, h1, l1;
    split_bf16(acc[2 * e], h0, l0);
    split_bf16(acc[2 * e + 1], h1, l1);
    oh[e] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
    ol[e] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
  }
  *reinterpret_cast<uint4*>(yh + opix * ys + y_off + g * 8) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
  *reinterpret_cast<uint4*>(yl + opix * ys + y_off + g * 8) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
}

}  // namespace stp3

using namespace stp3;
typedef __nv_bfloat16 bf16;

extern "C" int stp3_f32_to_hilo(const float* x, int channels_last, int n_img, int C, int H, int W, int cp, void* hi,
                                void* lo, void* stream) {
  STP3_CHECK_ARG(x && hi && lo && n_img > 0 && C > 0 && H > 0 && W > 0 && cp >= C, "stp3_f32_to_hilo: bad argument");
  const int HW = H * W;
  dim3 grid(ceil_div(HW, 32), ceil_div(cp, 32), n_img), block(32, 8);
  f32_to_hilo_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, channels_last, C, HW, cp, (bf16*)hi, (bf16*)lo);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_hilo_to_f32(const void* hi, const void* lo, int n_img, int H, int W, int cstride, int c_off, int C,
                                float* out, void* stream) {
  STP3_CHECK_ARG(hi && lo && out && n_img > 0 && C > 0 && c_off >= 0 && c_off + C <= cstride, "stp3_hilo_to_f32: bad argument");
  const int HW = H * W;
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), n_img), block(32, 8);
  hilo_to_f32_kernel<<<grid, block, 0, (cudaStream_t)stream>>>((const bf16*)hi, (const bf16*)lo, cstride, c_off, C, HW, out);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_spatial_sum(const void* hi, const void* lo, int n_img, int HW, int cstride, float* sums, void* stream) {
  STP3_CHECK_ARG(hi && lo && sums && n_img > 0 && HW > 0 && cstride > 0 && cstride <= 1024, "stp3_spatial_sum: bad argument");
  STP3_CUDA_OK(cudaMemsetAsync(sums, 0, (size_t)n_img * cstride * sizeof(float), (cudaStream_t)stream));
  const int px_per_block = 128;
  dim3 grid(ceil_div(HW, px_per_block), n_img);
  spatial_sum_kernel<<<grid, cstride, 0, (cudaStream_t)stream>>>((const bf16*)hi, (const bf16*)lo, HW, cstride, px_per_block, sums);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_pool_bias(const float* sums, int sums_stride, int n_img, int T, int C, float inv_hw, int temporal,
                              const float* const_vals, int n_const,
                              const float* W1, const float* b1, int R, const float* W2, int CO, const float* bias,
                              float* out, int co_stride, int accumulate, void* stream) {
  STP3_CHECK_ARG(sums && W1 && b1 && W2 && out && n_img > 0 && T > 0 && C > 0 && R > 0 && CO > 0 && n_const >= 0 &&
                 n_const < C && C - n_const <= sums_stride && CO <= co_stride && (n_const == 0 || const_vals),
                 "stp3_pool_bias: bad argument");
  STP3_CUDA_OK(launch_pdl(pool_bias_kernel, dim3(n_img, CO >= 64 ? 4 : 1), dim3(256), (size_t)(C + R) * sizeof(float), (cudaStream_t)stream,
                          sums, sums_stride, T, C, inv_hw, temporal, const_vals, n_const, W1, b1, R, W2, CO, bias, out,
                          co_stride, accumulate));
  return STP3_OK;
}

extern "C" int stp3_small_linear(const float* x, const float* W, int n, int ci, int co, const float* bias, float* y,
                                 int co_stride, int accumulate, void* stream) {
  STP3_CHECK_ARG(x && W && y && n > 0 && ci > 0 && co > 0 && co <= co_stride, "stp3_small_linear: bad argument");
  STP3_CUDA_OK(launch_pdl(small_linear_kernel, dim3(n), dim3(128), 0, (cudaStream_t)stream, x, W, ci, co, bias, y,
                          co_stride, accumulate));
  return STP3_OK;
}

extern "C" int stp3_upsample2x_add(const void* x_hi, const void* x_lo, int n_img, int h, int w, int x_cstride,
                                   const void* s_hi, const void* s_lo, int s_cstride, int s_coff, void* y_hi, void* y_lo,
                                   int y_cstride, int y_coff, int C, void* stream) {
  STP3_CHECK_ARG(x_hi && x_lo && y_hi && y_lo && n_img > 0 && h > 0 && w > 0, "stp3_upsample2x_add: null/empty");
  STP3_CHECK_ARG((s_hi == nullptr) == (s_lo == nullptr), "stp3_upsample2x_add: give both skip planes or neither");
  if (!s_hi) { s_cstride = 8; s_coff = 0; }
  STP3_CHECK_ARG(C % 8 == 0 && C <= x_cstride && s_coff % 8 == 0 && (!s_hi || s_coff + C <= s_cstride) &&
                 y_coff % 8 == 0 && y_coff + C <= y_cstride && x_cstride % 8 == 0 && s_cstride % 8 == 0 &&
                 y_cstride % 8 == 0, "stp3_upsample2x_add: channel windows must be multiples of 8");
  const size_t total = (size_t)n_img * (2 * h) * (2 * w) * (C / 8);
    STP3_CUDA_OK(launch_pdl(upsample2x_add_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream,
      (const bf16*)x_hi, (const bf16*)x_lo, h, w, x_cstride, (const bf16*)s_hi, (const bf16*)s_lo, s_cstride, s_coff,
      (bf16*)y_hi, (bf16*)y_lo, y_cstride, y_coff, C / 8, total));
  return STP3_OK;
}
