// Memory-bound per-pixel kernels of the eval-mode prediction stage (present distribution, Dual_GRU, SpatialGRU,
// ConvNeXt Block, Bottleblock): GRU gating, LayerNorm / GELU, depthwise 7x7 + LayerNorm, the trusting-gate softmax mix,
// the Bottleneck skip's pad-then-maxpool, and slot copies / broadcasts.  The convolutions themselves run on
// stp3_conv_fwd.  Every tensor is a channels-last bf16 hi/lo plane addressed through an stp3_hl_slot; every lane owns
// 8 consecutive channels of one pixel (one 128-bit load per plane), a pixel's lanes reduce with shuffles in a fixed
// order, and nothing is accumulated with atomics, so every result is a pure function of the inputs.
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace stp3 {
namespace {

struct Slot {
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
  int cstride, coff, t_total, t0;
};

// first element of pixel `pix` of call image `img` (of T frames per sample) in the slot
__device__ __forceinline__ size_t slot_index(const Slot& s, int img, int T, long long HW, long long pix) {
  const long long frame = (long long)(img / T) * s.t_total + s.t0 + img % T;
  return (size_t)((frame * HW + pix) * s.cstride + s.coff);
}

__device__ __forceinline__ void load8(const Slot& s, size_t i, float v[8]) {
  const uint4 h = *reinterpret_cast<const uint4*>(s.hi + i);
  const uint4 l = *reinterpret_cast<const uint4*>(s.lo + i);
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = ptx::join_hilo(hw[k], lw[k]);
    v[2 * k] = f.x;
    v[2 * k + 1] = f.y;
  }
}

__device__ __forceinline__ void store8(const Slot& s, size_t i, const float v[8]) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) ptx::split_hilo(v[2 * k], v[2 * k + 1], hw[k], lw[k]);
  *reinterpret_cast<uint4*>(s.hi + i) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  *reinterpret_cast<uint4*>(s.lo + i) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

// Sum over the L lanes of a pixel (L a power of two <= 32, the pixel's lanes contiguous within the warp); every lane
// of the warp must call it.  The butterfly adds in the same order for every pixel and launch.
template <int L>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, L);
  return v;
}

// Thread -> (pixel, lane) with L lanes per pixel; `valid` is false for the tail threads and the lanes beyond C / 8
struct Lane {
  long long p;        // pixel over all images: img * HW + pix
  int c;              // first of the lane's 8 channels
  bool pix_ok, valid;
};

template <int L>
__device__ __forceinline__ Lane lane_of(long long n_pix, int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  Lane r;
  r.p = t / L;
  r.c = (int)(t % L) * 8;
  r.pix_ok = r.p < n_pix;
  r.valid = r.pix_ok && r.c < C;
  return r;
}

// out = (1 - sigmoid(r)) * h
__global__ void __launch_bounds__(256)
gru_gates_kernel(Slot r, Slot h, Slot out, int T, long long HW, long long n_pix, int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = C / 8;
  if (t >= n_pix * cg) return;
  const long long p = t / cg;
  const int c = (int)(t % cg) * 8;
  const int img = (int)(p / HW);
  const long long pix = p % HW;
  float rv[8], hv[8];
  load8(r, slot_index(r, img, T, HW, pix) + c, rv);
  load8(h, slot_index(h, img, T, HW, pix) + c, hv);
#pragma unroll
  for (int k = 0; k < 8; ++k) rv[k] = (1.f - sigmoid_f(rv[k])) * hv[k];
  store8(out, slot_index(out, img, T, HW, pix) + c, rv);
}

// out (and out2) = (1 - sigmoid(u)) * h + sigmoid(u) * h_tilde; out may be h itself (each lane reads before it writes)
__global__ void __launch_bounds__(256)
gru_update_kernel(Slot u, Slot h, Slot ht, Slot out, Slot out2, int has_out2, int T, long long HW, long long n_pix,
                  int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = C / 8;
  if (t >= n_pix * cg) return;
  const long long p = t / cg;
  const int c = (int)(t % cg) * 8;
  const int img = (int)(p / HW);
  const long long pix = p % HW;
  float uv[8], hv[8], tv[8];
  load8(u, slot_index(u, img, T, HW, pix) + c, uv);
  load8(h, slot_index(h, img, T, HW, pix) + c, hv);
  load8(ht, slot_index(ht, img, T, HW, pix) + c, tv);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float g = sigmoid_f(uv[k]);
    uv[k] = (1.f - g) * hv[k] + g * tv[k];
  }
  store8(out, slot_index(out, img, T, HW, pix) + c, uv);
  if (has_out2) store8(out2, slot_index(out2, img, T, HW, pix) + c, uv);
}

// LayerNorm over the C channels of one pixel (biased variance, two passes over the registers)
template <int L>
__device__ __forceinline__ void layer_norm8(float v[8], bool valid, int c, int C, const float* gamma,
                                            const float* beta, float eps) {
  float s = 0.f;
  if (valid) {
#pragma unroll
    for (int k = 0; k < 8; ++k) s += v[k];
  }
  const float mean = group_sum<L>(s) / C;
  float q = 0.f;
  if (valid) {
#pragma unroll
    for (int k = 0; k < 8; ++k) q += (v[k] - mean) * (v[k] - mean);
  }
  const float inv = 1.f / sqrtf(group_sum<L>(q) / C + eps);
  if (valid) {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (v[k] - mean) * inv * gamma[c + k] + beta[c + k];
  }
}

// out = [gelu]([LN](x)) + [gelu](y)   (each bracket optional; no y: nothing added)
template <int L>
__global__ void __launch_bounds__(256)
channel_norm_act_kernel(Slot x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int gelu,
                        Slot y, int has_y, int gelu_y, Slot out, int T, long long HW, long long n_pix, int C) {
  const Lane ln = lane_of<L>(n_pix, C);
  const int img = ln.pix_ok ? (int)(ln.p / HW) : 0;
  const long long pix = ln.pix_ok ? ln.p % HW : 0;
  float v[8];
  if (ln.valid) load8(x, slot_index(x, img, T, HW, pix) + ln.c, v);
  if (gamma != nullptr) layer_norm8<L>(v, ln.valid, ln.c, C, gamma, beta, eps);
  if (!ln.valid) return;
  if (gelu) {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = gelu_f(v[k]);
  }
  if (has_y) {
    float w[8];
    load8(y, slot_index(y, img, T, HW, pix) + ln.c, w);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] += gelu_y ? gelu_f(w[k]) : w[k];
  }
  store8(out, slot_index(out, img, T, HW, pix) + ln.c, v);
}

// out = LN(depthwise k x k (zero padding k/2) of x + bias)
template <int L>
__global__ void __launch_bounds__(256)
dw_ln_kernel(Slot x, const float* __restrict__ w, const float* __restrict__ bias, int k, const float* __restrict__ gamma,
             const float* __restrict__ beta, float eps, Slot out, int T, int H, int W, long long n_pix, int C) {
  const long long HW = (long long)H * W;
  const Lane ln = lane_of<L>(n_pix, C);
  const int img = ln.pix_ok ? (int)(ln.p / HW) : 0;
  const long long pix = ln.pix_ok ? ln.p % HW : 0;
  const int py = (int)(pix / W), px = (int)(pix % W);
  float v[8];
  if (ln.valid) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = bias[ln.c + j];
    const size_t base = slot_index(x, img, T, HW, 0) + ln.c;
    const int pad = k / 2;
    for (int ky = 0; ky < k; ++ky) {
      const int iy = py + ky - pad;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < k; ++kx) {
        const int ix = px + kx - pad;
        if (ix < 0 || ix >= W) continue;
        float a[8];
        load8(x, base + ((size_t)iy * W + ix) * x.cstride, a);
        const float4 w0 = *reinterpret_cast<const float4*>(w + (size_t)(ky * k + kx) * C + ln.c);
        const float4 w1 = *reinterpret_cast<const float4*>(w + (size_t)(ky * k + kx) * C + ln.c + 4);
        v[0] = fmaf(a[0], w0.x, v[0]); v[1] = fmaf(a[1], w0.y, v[1]);
        v[2] = fmaf(a[2], w0.z, v[2]); v[3] = fmaf(a[3], w0.w, v[3]);
        v[4] = fmaf(a[4], w1.x, v[4]); v[5] = fmaf(a[5], w1.y, v[5]);
        v[6] = fmaf(a[6], w1.z, v[6]); v[7] = fmaf(a[7], w1.w, v[7]);
      }
    }
  }
  layer_norm8<L>(v, ln.valid, ln.c, C, gamma, beta, eps);
  if (ln.valid) store8(out, slot_index(out, img, T, HW, pix) + ln.c, v);
}

constexpr int kMaxMixDst = 4;
struct MixDst {
  Slot d[kMaxMixDst];
};

// z = W t (W (2, C)), p = softmax(z), mix = s2 * p0 + s1 * p1 written to every destination
template <int L>
__global__ void __launch_bounds__(256)
trust_mix_kernel(Slot t_in, const float* __restrict__ w, Slot s1, Slot s2, MixDst dst, int n_dst, int T, long long HW,
                 long long n_pix, int C) {
  const Lane ln = lane_of<L>(n_pix, C);
  const int img = ln.pix_ok ? (int)(ln.p / HW) : 0;
  const long long pix = ln.pix_ok ? ln.p % HW : 0;
  float z0 = 0.f, z1 = 0.f;
  if (ln.valid) {
    float v[8];
    load8(t_in, slot_index(t_in, img, T, HW, pix) + ln.c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      z0 = fmaf(w[ln.c + k], v[k], z0);
      z1 = fmaf(w[C + ln.c + k], v[k], z1);
    }
  }
  z0 = group_sum<L>(z0);
  z1 = group_sum<L>(z1);
  if (!ln.valid) return;
  const float m = fmaxf(z0, z1);
  const float e0 = expf(z0 - m), e1 = expf(z1 - m);
  const float p0 = e0 / (e0 + e1), p1 = e1 / (e0 + e1);
  float a[8], b[8];
  load8(s1, slot_index(s1, img, T, HW, pix) + ln.c, a);
  load8(s2, slot_index(s2, img, T, HW, pix) + ln.c, b);
#pragma unroll
  for (int k = 0; k < 8; ++k) a[k] = b[k] * p0 + a[k] * p1;
#pragma unroll
  for (int i = 0; i < kMaxMixDst; ++i)
    if (i < n_dst) store8(dst.d[i], slot_index(dst.d[i], img, T, HW, pix) + ln.c, a);
}

// out (ceil(H/2), ceil(W/2)) = 2x2 max of x zero-padded by one row / column where H / W is odd.  The winner's hi / lo
// bits are stored as they are (a padded zero as +0 / +0), so the result is exact.
__global__ void __launch_bounds__(256)
maxpool2_pad_kernel(Slot x, Slot out, int T, int H, int W, long long n_pix_out, int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = C / 8;
  if (t >= n_pix_out * cg) return;
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long HWo = (long long)Ho * Wo, HW = (long long)H * W;
  const long long p = t / cg;
  const int c = (int)(t % cg) * 8;
  const int img = (int)(p / HWo);
  const int oy = (int)(p % HWo / Wo), ox = (int)(p % Wo);
  float m[8];
  alignas(16) uint16_t mh[8], ml[8];
  const size_t base = slot_index(x, img, T, HW, 0) + c;
  for (int d = 0; d < 4; ++d) {
    const int iy = 2 * oy + (d >> 1), ix = 2 * ox + (d & 1);
    alignas(16) uint16_t vh[8] = {0, 0, 0, 0, 0, 0, 0, 0}, vl[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (iy < H && ix < W) {
      const size_t i = base + ((size_t)iy * W + ix) * x.cstride;
      *reinterpret_cast<uint4*>(vh) = *reinterpret_cast<const uint4*>(x.hi + i);
      *reinterpret_cast<uint4*>(vl) = *reinterpret_cast<const uint4*>(x.lo + i);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float v = __uint_as_float((uint32_t)vh[k] << 16) + __uint_as_float((uint32_t)vl[k] << 16);
      if (d == 0 || v > m[k]) {
        m[k] = v;
        mh[k] = vh[k];
        ml[k] = vl[k];
      }
    }
  }
  const size_t o = slot_index(out, img, T, HWo, (long long)oy * Wo + ox) + c;
  *reinterpret_cast<uint4*>(out.hi + o) = *reinterpret_cast<const uint4*>(mh);
  *reinterpret_cast<uint4*>(out.lo + o) = *reinterpret_cast<const uint4*>(ml);
}

// out = x (channel slot to channel slot, bit for bit), or out = vec[img] at every pixel
__global__ void __launch_bounds__(256)
hl_copy_kernel(Slot src, const float* __restrict__ vec, int vstride, Slot dst, int T, long long HW, long long n_pix,
               int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = C / 8;
  if (t >= n_pix * cg) return;
  const long long p = t / cg;
  const int c = (int)(t % cg) * 8;
  const int img = (int)(p / HW);
  const long long pix = p % HW;
  const size_t o = slot_index(dst, img, T, HW, pix) + c;
  if (vec != nullptr) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = vec[(size_t)img * vstride + c + k];
    store8(dst, o, v);
  } else {           // bit copy of both planes
    const size_t i = slot_index(src, img, T, HW, pix) + c;
    *reinterpret_cast<uint4*>(dst.hi + o) = *reinterpret_cast<const uint4*>(src.hi + i);
    *reinterpret_cast<uint4*>(dst.lo + o) = *reinterpret_cast<const uint4*>(src.lo + i);
  }
}

// ------------------------------------------------------------------------------------------------ host side
int to_slot(const char* fn, const char* name, const stp3_hl_slot* s, int T, int C, Slot& out) {
  STP3_CHECK_ARG(s != nullptr && s->hi != nullptr && s->lo != nullptr, "%s: %s is null", fn, name);
  STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(s->hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(s->lo) & 15) == 0,
                 "%s: %s planes must be 16-byte aligned", fn, name);
  STP3_CHECK_ARG(s->cstride > 0 && s->cstride % 8 == 0 && s->coff >= 0 && s->coff % 8 == 0 && s->coff + C <= s->cstride,
                 "%s: %s channels [%d, %d) do not fit a multiple-of-8 slot of a %d-channel stride", fn, name, s->coff,
                 s->coff + C, s->cstride);
  STP3_CHECK_ARG(s->t0 >= 0 && s->t0 + T <= s->t_total, "%s: %s frames [%d, %d) outside its %d frames", fn, name, s->t0,
                 s->t0 + T, s->t_total);
  out = Slot{static_cast<__nv_bfloat16*>(s->hi), static_cast<__nv_bfloat16*>(s->lo), s->cstride, s->coff, s->t_total,
             s->t0};
  return STP3_OK;
}

// The element range [first, last) a slot spans in each plane over B samples of T frames of HW pixels
inline void slot_span(const Slot& s, int B, int T, long long HW, const __nv_bfloat16* base, uintptr_t& lo,
                      uintptr_t& hi) {
  const long long first = (long long)s.t0 * HW * s.cstride;
  const long long last = ((long long)(B - 1) * s.t_total + s.t0 + T) * HW * s.cstride;
  lo = reinterpret_cast<uintptr_t>(base + first);
  hi = reinterpret_cast<uintptr_t>(base + last);
}

// true when any plane of a overlaps any plane of b (their spans, conservatively: channel slots are not told apart)
inline bool slots_overlap(const Slot& a, const Slot& b, int B, int T, long long HW) {
  const __nv_bfloat16* pa[2] = {a.hi, a.lo};
  const __nv_bfloat16* pb[2] = {b.hi, b.lo};
  for (const __nv_bfloat16* x : pa) {
    for (const __nv_bfloat16* y : pb) {
      uintptr_t x0, x1, y0, y1;
      slot_span(a, B, T, HW, x, x0, x1);
      slot_span(b, B, T, HW, y, y0, y1);
      if (x0 < y1 && y0 < x1) return true;
    }
  }
  return false;
}

int check_dims(const char* fn, int B, int T, long long HW, int C, int c_max) {
  STP3_CHECK_ARG(B >= 0 && T > 0 && HW >= 0, "%s: bad shape B=%d T=%d HW=%lld", fn, B, T, HW);
  STP3_CHECK_ARG(C > 0 && C % 8 == 0 && C <= c_max, "%s: C = %d must be a positive multiple of 8 <= %d", fn, C, c_max);
  return STP3_OK;
}

#define STP3_TRY(expr)          \
  do {                          \
    const int rc__ = (expr);    \
    if (rc__ != STP3_OK) return rc__; \
  } while (0)

inline unsigned blocks_for(long long threads) { return (unsigned)((threads + 255) / 256); }

// lanes per pixel of the reducing kernels: the power of two that holds C / 8
inline int lanes_for(int C) {
  int L = 1;
  while (L * 8 < C) L *= 2;
  return L;
}

template <template <int> class K, typename... Args>
cudaError_t launch_lanes(int C, long long n_pix, cudaStream_t st, Args... args) {
  const int L = lanes_for(C);
  const unsigned g = blocks_for(n_pix * L);
  switch (L) {
    case 1: K<1>::run(g, st, args...); break;
    case 2: K<2>::run(g, st, args...); break;
    case 4: K<4>::run(g, st, args...); break;
    case 8: K<8>::run(g, st, args...); break;
    case 16: K<16>::run(g, st, args...); break;
    default: K<32>::run(g, st, args...); break;
  }
  return cudaGetLastError();
}

template <int L>
struct NormAct {
  template <typename... A>
  static void run(unsigned g, cudaStream_t st, A... a) { channel_norm_act_kernel<L><<<g, 256, 0, st>>>(a...); }
};
template <int L>
struct DwLn {
  template <typename... A>
  static void run(unsigned g, cudaStream_t st, A... a) { dw_ln_kernel<L><<<g, 256, 0, st>>>(a...); }
};
template <int L>
struct TrustMix {
  template <typename... A>
  static void run(unsigned g, cudaStream_t st, A... a) { trust_mix_kernel<L><<<g, 256, 0, st>>>(a...); }
};

}  // namespace
}  // namespace stp3

using namespace stp3;

extern "C" int stp3_gru_gates(const stp3_hl_slot* r, const stp3_hl_slot* h, const stp3_hl_slot* out, int B, int T,
                              long long HW, int C, void* stream) {
  const char* fn = "stp3_gru_gates";
  STP3_TRY(check_dims(fn, B, T, HW, C, 1 << 20));
  Slot R, H, O;
  STP3_TRY(to_slot(fn, "r", r, T, C, R));
  STP3_TRY(to_slot(fn, "h", h, T, C, H));
  STP3_TRY(to_slot(fn, "out", out, T, C, O));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  gru_gates_kernel<<<blocks_for(n_pix * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(R, H, O, T, HW, n_pix, C);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_gru_update(const stp3_hl_slot* u, const stp3_hl_slot* h, const stp3_hl_slot* h_tilde,
                               const stp3_hl_slot* out, const stp3_hl_slot* out2, int B, int T, long long HW, int C,
                               void* stream) {
  const char* fn = "stp3_gru_update";
  STP3_TRY(check_dims(fn, B, T, HW, C, 1 << 20));
  Slot U, H, Ht, O, O2{};
  STP3_TRY(to_slot(fn, "u", u, T, C, U));
  STP3_TRY(to_slot(fn, "h", h, T, C, H));
  STP3_TRY(to_slot(fn, "h_tilde", h_tilde, T, C, Ht));
  STP3_TRY(to_slot(fn, "out", out, T, C, O));
  if (out2 != nullptr) STP3_TRY(to_slot(fn, "out2", out2, T, C, O2));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  gru_update_kernel<<<blocks_for(n_pix * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      U, H, Ht, O, O2, out2 != nullptr, T, HW, n_pix, C);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_channel_norm_act(const stp3_hl_slot* x, const float* gamma, const float* beta, float eps, int gelu,
                                     const stp3_hl_slot* y, int gelu_y, const stp3_hl_slot* out, int B, int T,
                                     long long HW, int C, void* stream) {
  const char* fn = "stp3_channel_norm_act";
  STP3_TRY(check_dims(fn, B, T, HW, C, 256));
  STP3_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "%s: gamma and beta are given together or not at all", fn);
  STP3_CHECK_ARG(gamma == nullptr || eps > 0.f, "%s: eps must be positive", fn);
  Slot X, Y{}, O;
  STP3_TRY(to_slot(fn, "x", x, T, C, X));
  if (y != nullptr) STP3_TRY(to_slot(fn, "y", y, T, C, Y));
  STP3_TRY(to_slot(fn, "out", out, T, C, O));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  STP3_CUDA_OK((launch_lanes<NormAct>(C, n_pix, static_cast<cudaStream_t>(stream), X, gamma, beta, eps, gelu, Y,
                                      int(y != nullptr), gelu_y, O, T, HW, n_pix, C)));
  return STP3_OK;
}

extern "C" int stp3_dw_ln(const stp3_hl_slot* x, const float* w, const float* bias, int k, const float* gamma,
                          const float* beta, float eps, const stp3_hl_slot* out, int B, int T, int H, int W, int C,
                          void* stream) {
  const char* fn = "stp3_dw_ln";
  STP3_CHECK_ARG(H >= 0 && W >= 0, "%s: bad map %dx%d", fn, H, W);
  STP3_TRY(check_dims(fn, B, T, (long long)H * W, C, 256));
  STP3_CHECK_ARG(k > 0 && k % 2 == 1 && k <= 15, "%s: k = %d must be odd and <= 15", fn, k);
  STP3_CHECK_ARG(w != nullptr && bias != nullptr && gamma != nullptr && beta != nullptr, "%s: null parameter", fn);
  STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(w) & 15) == 0, "%s: w must be 16-byte aligned", fn);
  STP3_CHECK_ARG(eps > 0.f, "%s: eps must be positive", fn);
  Slot X, O;
  STP3_TRY(to_slot(fn, "x", x, T, C, X));
  STP3_TRY(to_slot(fn, "out", out, T, C, O));
  STP3_CHECK_ARG(!slots_overlap(X, O, B, T, (long long)H * W), "%s: out's planes overlap x's (every tap reads "
                 "neighbouring pixels another thread may already have written)", fn);
  const long long n_pix = (long long)B * T * H * W;
  if (n_pix == 0) return STP3_OK;
  STP3_CUDA_OK((launch_lanes<DwLn>(C, n_pix, static_cast<cudaStream_t>(stream), X, w, bias, k, gamma, beta, eps, O, T,
                                   H, W, n_pix, C)));
  return STP3_OK;
}

extern "C" int stp3_trust_mix(const stp3_hl_slot* t, const float* w, const stp3_hl_slot* s1, const stp3_hl_slot* s2,
                              const stp3_hl_slot* dst, int n_dst, int B, int T, long long HW, int C, void* stream) {
  const char* fn = "stp3_trust_mix";
  STP3_TRY(check_dims(fn, B, T, HW, C, 256));
  STP3_CHECK_ARG(w != nullptr, "%s: w is null", fn);
  STP3_CHECK_ARG(dst != nullptr && n_dst >= 1 && n_dst <= kMaxMixDst, "%s: 1 to %d destinations, got %d", fn,
                 kMaxMixDst, n_dst);
  Slot Tt, S1, S2;
  MixDst D{};
  STP3_TRY(to_slot(fn, "t", t, T, C, Tt));
  STP3_TRY(to_slot(fn, "s1", s1, T, C, S1));
  STP3_TRY(to_slot(fn, "s2", s2, T, C, S2));
  for (int i = 0; i < n_dst; ++i) STP3_TRY(to_slot(fn, "dst", dst + i, T, C, D.d[i]));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  STP3_CUDA_OK((launch_lanes<TrustMix>(C, n_pix, static_cast<cudaStream_t>(stream), Tt, w, S1, S2, D, n_dst, T, HW,
                                       n_pix, C)));
  return STP3_OK;
}

extern "C" int stp3_maxpool2_pad(const stp3_hl_slot* x, const stp3_hl_slot* out, int B, int T, int H, int W, int C,
                                 void* stream) {
  const char* fn = "stp3_maxpool2_pad";
  STP3_CHECK_ARG(H >= 0 && W >= 0, "%s: bad map %dx%d", fn, H, W);
  STP3_TRY(check_dims(fn, B, T, (long long)H * W, C, 1 << 20));
  Slot X, O;
  STP3_TRY(to_slot(fn, "x", x, T, C, X));
  STP3_TRY(to_slot(fn, "out", out, T, C, O));
  const long long n_out = (long long)B * T * ((H + 1) / 2) * ((W + 1) / 2);
  if (n_out == 0) return STP3_OK;
  maxpool2_pad_kernel<<<blocks_for(n_out * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(X, O, T, H, W, n_out,
                                                                                                  C);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_hl_copy(const stp3_hl_slot* src, const stp3_hl_slot* dst, int B, int T, long long HW, int C,
                            void* stream) {
  const char* fn = "stp3_hl_copy";
  STP3_TRY(check_dims(fn, B, T, HW, C, 1 << 20));
  Slot S, D;
  STP3_TRY(to_slot(fn, "src", src, T, C, S));
  STP3_TRY(to_slot(fn, "dst", dst, T, C, D));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  hl_copy_kernel<<<blocks_for(n_pix * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(S, nullptr, 0, D, T, HW,
                                                                                              n_pix, C);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_hl_broadcast(const float* vec, int vstride, const stp3_hl_slot* dst, int B, int T, long long HW,
                                 int C, void* stream) {
  const char* fn = "stp3_hl_broadcast";
  STP3_TRY(check_dims(fn, B, T, HW, C, 1 << 20));
  STP3_CHECK_ARG(vec != nullptr && vstride >= C, "%s: vec is null or its row stride %d < C = %d", fn, vstride, C);
  Slot D;
  STP3_TRY(to_slot(fn, "dst", dst, T, C, D));
  const long long n_pix = (long long)B * T * HW;
  if (n_pix == 0) return STP3_OK;
  hl_copy_kernel<<<blocks_for(n_pix * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(D, vec, vstride, D, T, HW,
                                                                                              n_pix, C);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
