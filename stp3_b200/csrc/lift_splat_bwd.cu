// Backward of the fused lift-splat (SURVEY.md row f2): gradients of the BEV features with respect to the context
// features and the depth logits, i.e. the autograd chain the reference trains through --
//   VoxelsSumming.backward (stp3/utils/geometry.py:321-330: every point receives the gradient of its pillar),
//   the mask / sort / index_put of projection_to_birds_eye_view (stp3.py:239-296; the discount recurrence
//   bev = bev * discount + tmp makes frame t' feed every output frame t >= t' with weight discount^(t - t')),
//   the outer product and the softmax over depth of encoder_forward (stp3.py:214-216).
// The voxel indices are not differentiable (integer) and are recomputed with the forward's exact arithmetic
// (lift_geom.cuh), so forward and backward agree on every point's pillar.
//
//   K1  bev_grad_to_grid_kernel : g_grid[b,t',pillar,c] = sum_{t >= t'} discount^(t-t') * g_out[b,t,c,pillar]
//         (channels-last, so that a point's gradient row is one contiguous 4*C-byte gather)
//   K2  lift_splat_bwd_kernel   : one CTA per (b, t, camera, 4 image columns), one warp per column, lanes = channel pairs
//         (one body for both feature layouts: NCHW, and channels-last -- what the encoder heads produce -- where a
//          lane's channel pair is one float2 of a pixel's contiguous row; only the addresses of feat / g_feat differ,
//          every sum keeps its order, so the two instantiations agree bit for bit)
//         g_feat[c,h,w]  = sum_d prob[d,h,w] * g_grid[rank(d,h,w), c]
//         g_prob[d,h,w]  = sum_c feat[c,h,w] * g_grid[rank(d,h,w), c]      (halving butterfly over the lanes)
//         g_logit[d,h,w] = prob[d,h,w] * (g_prob[d,h,w] - sum_d' prob[d',h,w] * g_prob[d',h,w])
// Gathers only -- no atomics: deterministic.
#include <cmath>
#include <cstdint>

#include "common.cuh"
#include "lift_geom.cuh"

namespace stp3 {

constexpr int kBwdTW = 4;            // image columns per CTA = warps per CTA
constexpr int kBwdH = 16;            // image rows whose feature / gradient accumulators a lane keeps in registers
constexpr int kBwdC = 64;            // channels per pass (2 per lane)
constexpr int kBwdMaxFrames = 8;

struct LiftBwdParams {
  const float* feat;      // (B,S,N,C,Hf,Wf), channels-last instantiation: (B,S,N,Hf,Wf,C)
  const float* depth;     // (B,S,N,D,Hf,Wf) or null
  const float* cam_M; const float* cam_t; const float* ego_R; const float* ego_t;
  const float* xs; const float* ys; const float* ds;
  BevQuant q;
  int B, S, N, D, Hf, Wf, C;
  int use_depth;
  int tiles_w;
  const float* ggrid;     // (B,S,nvox,C)
  float* gfeat;           // same layout as feat
  float* gdepth;          // (B,S,N,D,Hf,Wf) or null
};

// g_grid[b,t',v,c] = g_out[b,t',c,v] + discount * g_grid[b,t'+1,v,c]: tile of 32 pillars x 32 channels through shared
// memory (reads coalesced along pillars, writes along channels)
__global__ void __launch_bounds__(256)
bev_grad_to_grid_kernel(const float* __restrict__ gout, float* __restrict__ ggrid, int S, int C, int nvox, float discount) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, v0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};          // thread (x, y) carries channels c0 + y + 8*i of pillar v0 + x
  for (int t = S - 1; t >= 0; --t) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + threadIdx.y + 8 * i, v = v0 + threadIdx.x;
      const float g = (c < C && v < nvox) ? gout[(((size_t)b * S + t) * C + c) * nvox + v] : 0.f;
      acc[i] = __fadd_rn(__fmul_rn(acc[i], discount), g);
      tile[threadIdx.y + 8 * i][threadIdx.x] = acc[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int v = v0 + threadIdx.y + 8 * i, c = c0 + threadIdx.x;
      if (c < C && v < nvox) ggrid[(((size_t)b * S + t) * nvox + v) * C + c] = tile[threadIdx.x][threadIdx.y + 8 * i];
    }
    __syncthreads();
  }
}

template <bool kChannelsLast>
__global__ void __launch_bounds__(32 * kBwdTW, 2)
lift_splat_bwd_kernel(const LiftBwdParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int TW = kBwdTW;
  const int D = p.D, Hf = p.Hf, Wf = p.Wf, C = p.C;
  const int npix = Hf * TW;
  const int fstride = npix | 1;                                        // odd row stride: conflict-free register fills
  float* s_prob = reinterpret_cast<float*>(smem_raw);                  // [D][TW][Hf] softmax(depth), NOT masked
  int* s_rank = reinterpret_cast<int*>(s_prob + D * npix);             // [D][TW][Hf]
  float* s_gp = reinterpret_cast<float*>(s_rank + D * npix);           // [D][TW][Hf] gradient w.r.t. the probability
  float* s_feat = s_gp + D * npix;                                     // [64][fstride]
  float* s_mat = s_feat + kBwdC * fstride;                             // camera 12 + chain 12 * (kBwdMaxFrames - 1)
  float* s_ys = s_mat + 12 * kBwdMaxFrames;
  float* s_ds = s_ys + Hf;

  const int tid = threadIdx.x, nthr = blockDim.x;
  int blk = blockIdx.x;
  const int tile = blk % p.tiles_w; blk /= p.tiles_w;
  const int n = blk % p.N; blk /= p.N;
  const int frame = blk;                         // b*S + t
  const int t = frame % p.S, b = frame / p.S;
  const int w0 = tile * TW;
  const int img = frame * p.N + n;
  const int n_chain = p.S - 1 - t;
  const size_t nvox = (size_t)p.q.nx * p.q.ny * p.q.nz;
  const float* gbase = p.ggrid + (size_t)frame * nvox * C;

  if (tid < 9) s_mat[tid] = p.cam_M[img * 9 + tid];
  if (tid >= 9 && tid < 12) s_mat[tid] = p.cam_t[img * 3 + tid - 9];
  for (int i = tid; i < n_chain * 12; i += nthr) {
    const int k = i / 12, e = i % 12;
    const int src = b * p.S + t + k;
    s_mat[12 + i] = e < 9 ? p.ego_R[src * 9 + e] : p.ego_t[src * 3 + e - 9];
  }
  for (int i = tid; i < Hf; i += nthr) s_ys[i] = p.ys[i];
  for (int i = tid; i < D; i += nthr) s_ds[i] = p.ds[i];
  __syncthreads();

  // ---- per pixel: softmax over D (stp3.py:215) and the rank of every point of its ray
  for (int px = tid; px < npix; px += nthr) {
    const int wl = px % TW, h = px / TW;
    const int w = w0 + wl;
    const bool inb = w < Wf;
    float* prow = s_prob + wl * Hf + h;            // + d * npix
    int* rrow = s_rank + wl * Hf + h;
    if (p.use_depth) {
      const float* dsrc = p.depth + ((size_t)img * D * Hf + h) * Wf + w;
      float mx = -INFINITY;
      for (int d = 0; d < D; ++d) {
        const float v = inb ? __ldg(dsrc + (size_t)d * Hf * Wf) : 0.f;
        prow[d * npix] = v;
        mx = fmaxf(mx, v);
      }
      float sum = 0.f;
      for (int d = 0; d < D; ++d) {
        const float e = __expf(prow[d * npix] - mx);
        prow[d * npix] = e;
        sum += e;
      }
      const float inv = __frcp_rn(sum);
      for (int d = 0; d < D; ++d) prow[d * npix] *= inv;
    } else {
      for (int d = 0; d < D; ++d) prow[d * npix] = 1.0f;
    }
    const float xw = inb ? __ldg(p.xs + w) : 0.f;
    const float yh = s_ys[h];
    for (int d = 0; d < D; ++d) {
      rrow[d * npix] = inb ? lifted_point_rank(p.q, s_mat, s_mat + 12, n_chain, xw, yh, s_ds[d]) : -1;
      s_gp[d * npix + wl * Hf + h] = 0.f;
    }
  }

  // ---- per channel pass: warp = image column, lane = channel pair
  const int warp = tid >> 5, lane = tid & 31;
  const int wl = warp, w = w0 + wl;
  for (int c0 = 0; c0 < C; c0 += kBwdC) {
    __syncthreads();
    if constexpr (kChannelsLast) {                                  // a warp reads one pixel's 64 channels: 256 contiguous bytes
      for (int i = tid; i < (kBwdC / 2) * npix; i += nthr) {
        const int l = i & 31, px = i >> 5;
        const int ww = w0 + px % TW, hh = px / TW;
        float2 v = make_float2(0.f, 0.f);
        if (ww < Wf && c0 + 2 * l < C)                              // C is even: the pair is inside together
          v = __ldg(reinterpret_cast<const float2*>(p.feat + (((size_t)img * Hf + hh) * Wf + ww) * C + c0 + 2 * l));
        s_feat[l * fstride + px] = v.x;
        s_feat[(l + 32) * fstride + px] = v.y;
      }
    } else {
      for (int i = tid; i < kBwdC * npix; i += nthr) {              // context features of channels [c0, c0+64) of the tile
        const int cl = i / npix, px = i % npix;
        const int ww = w0 + px % TW, hh = px / TW;
        float v = 0.f;
        if (ww < Wf && c0 + cl < C) v = __ldg(p.feat + (((size_t)img * C + c0 + cl) * Hf + hh) * Wf + ww);
        s_feat[(((cl & 1) << 5) | (cl >> 1)) * fstride + px] = v;   // channels (2l, 2l+1) in rows l and l + 32
      }
    }
    __syncthreads();
    if (w >= Wf) continue;
    const int c = c0 + 2 * lane;
    for (int h0 = 0; h0 < Hf; h0 += kBwdH) {
      float f0[kBwdH], f1[kBwdH], a0[kBwdH], a1[kBwdH];
#pragma unroll
      for (int j = 0; j < kBwdH; ++j) {
        const int h = h0 + j;
        f0[j] = h < Hf ? s_feat[lane * fstride + h * TW + wl] : 0.f;
        f1[j] = h < Hf ? s_feat[(lane + 32) * fstride + h * TW + wl] : 0.f;
        a0[j] = 0.f; a1[j] = 0.f;
      }
      for (int d = 0; d < D; ++d) {
        const int* rk = s_rank + d * npix + wl * Hf + h0;
        const float* pr = s_prob + d * npix + wl * Hf + h0;
        float part[kBwdH];
        int prev = -1;
        float g0 = 0.f, g1 = 0.f;
#pragma unroll
        for (int j = 0; j < kBwdH; ++j) {
          part[j] = 0.f;
          if (h0 + j < Hf) {
            const int r = rk[j];                                    // warp-uniform
            if (r >= 0) {
              if (r != prev) {                                      // neighbouring rows usually share the pillar
                g0 = 0.f; g1 = 0.f;
                if (c < C) {
                  const float* src = gbase + (size_t)r * C + c;
                  g0 = __ldg(src);
                  if (c + 1 < C) g1 = __ldg(src + 1);
                }
                prev = r;
              }
              const float q = pr[j];
              a0[j] = fmaf(q, g0, a0[j]);
              a1[j] = fmaf(q, g1, a1[j]);
              part[j] = fmaf(f0[j], g0, f1[j] * g1);
            }
          }
        }
        // sum the 32 lanes' partial dot products of the kBwdH points: halving butterfly, lane j ends with point j
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          const bool upper = (lane & off) != 0;
          if (off >= kBwdH) {                                       // more lanes than values left: plain pairwise sums
#pragma unroll
            for (int i = 0; i < kBwdH; ++i) part[i] += __shfl_xor_sync(0xffffffffu, part[i], off);
          } else {
#pragma unroll
            for (int i = 0; i < kBwdH / 2; ++i) {
              if (i < off) {
                const float send = upper ? part[i] : part[i + off];
                const float keep = upper ? part[i + off] : part[i];
                part[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
              }
            }
          }
        }
        // after the steps off = 8, 4, 2, 1 lane l holds in part[0] the sum for point (l & 15) (both halves of the
        // warp carry the same totals after the off = 16 step)
        if (lane < kBwdH && h0 + lane < Hf) s_gp[d * npix + wl * Hf + h0 + lane] += part[0];
        __syncwarp();
      }
#pragma unroll
      for (int j = 0; j < kBwdH; ++j) {
        const int h = h0 + j;
        if (h < Hf && c < C) {
          if constexpr (kChannelsLast) {
            *reinterpret_cast<float2*>(p.gfeat + (((size_t)img * Hf + h) * Wf + w) * C + c) = make_float2(a0[j], a1[j]);
          } else {
            p.gfeat[(((size_t)img * C + c) * Hf + h) * Wf + w] = a0[j];
            if (c + 1 < C) p.gfeat[(((size_t)img * C + c + 1) * Hf + h) * Wf + w] = a1[j];
          }
        }
      }
    }
  }
  __syncthreads();

  // ---- softmax backward per pixel
  if (p.gdepth && p.use_depth) {
    for (int px = tid; px < npix; px += nthr) {
      const int wl2 = px % TW, h = px / TW;
      const int w2 = w0 + wl2;
      if (w2 >= Wf) continue;
      const float* prow = s_prob + wl2 * Hf + h;
      const float* grow = s_gp + wl2 * Hf + h;
      float dot = 0.f;
      for (int d = 0; d < D; ++d) dot = fmaf(prow[d * npix], grow[d * npix], dot);
      float* dst = p.gdepth + ((size_t)img * D * Hf + h) * Wf + w2;
      for (int d = 0; d < D; ++d) dst[(size_t)d * Hf * Wf] = prow[d * npix] * (grow[d * npix] - dot);
    }
  }
}

}  // namespace stp3

using namespace stp3;

extern "C" size_t stp3_lift_splat_bwd_scratch_bytes(const stp3_lift_splat_desc* d) {
  if (!d || d->B <= 0 || d->S <= 0 || d->C <= 0 || d->nx <= 0 || d->ny <= 0) return 0;
  return (size_t)d->B * d->S * d->nx * d->ny * d->C * sizeof(float);
}

// Both entry points: the checks they share, K1, then K2 instantiated for the layout.  `fn` names the caller in messages.
template <bool kChannelsLast>
static int lift_splat_bwd_launch(const char* fn, const stp3_lift_splat_desc* desc, const float* grad_out, const float* feat,
                                 const float* depth_logits, void* scratch, size_t scratch_bytes, float* grad_feat,
                                 float* grad_depth_logits, cudaStream_t stream, LiftBwdParams& p) {
  STP3_CHECK_ARG(desc->f_count == 0, "%s: every frame is processed (f_count 0)", fn);
  const int B = desc->B, S = desc->S, N = desc->N, D = desc->D, Hf = desc->Hf, Wf = desc->Wf, C = desc->C;
  const size_t need = stp3_lift_splat_bwd_scratch_bytes(desc);
  if (scratch_bytes < need) return set_error(STP3_ENOSPC, "scratch too small: %zu < %zu", scratch_bytes, need);
  const int nvox = desc->nx * desc->ny * desc->nz;
  // every refusal comes before the first launch
  const int npix = Hf * kBwdTW;
  const size_t smem = ((size_t)3 * D * npix + (size_t)kBwdC * (npix | 1) + 12 * kBwdMaxFrames + Hf + D) * sizeof(float) + 16;
  STP3_CHECK_ARG(smem <= 227 * 1024, "D*Hf = %d too large for the backward tile in shared memory", D * Hf);
  const int tiles_w = ceil_div(Wf, kBwdTW);
  const long long nblk = (long long)B * S * N * tiles_w;
  STP3_CHECK_ARG(nblk < (1ll << 31), "grid too large");

  dim3 g1(ceil_div(nvox, 32), ceil_div(C, 32), B);
  bev_grad_to_grid_kernel<<<g1, dim3(32, 8), 0, stream>>>(grad_out, static_cast<float*>(scratch), S, C, nvox,
                                                          desc->discount);
  STP3_CUDA_OK(cudaGetLastError());

  p.feat = feat; p.depth = depth_logits; p.cam_M = desc->cam_M; p.cam_t = desc->cam_t; p.ego_R = desc->ego_R;
  p.ego_t = desc->ego_t; p.xs = desc->xs; p.ys = desc->ys; p.ds = desc->ds;
  p.B = B; p.S = S; p.N = N; p.D = D; p.Hf = Hf; p.Wf = Wf; p.C = C;
  p.use_depth = desc->use_depth_distribution;
  p.tiles_w = tiles_w;
  p.ggrid = static_cast<const float*>(scratch);
  p.gfeat = grad_feat; p.gdepth = grad_depth_logits;
  STP3_CUDA_OK(cudaFuncSetAttribute(lift_splat_bwd_kernel<kChannelsLast>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem));
  lift_splat_bwd_kernel<kChannelsLast><<<(unsigned)nblk, 32 * kBwdTW, smem, stream>>>(p);
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}

extern "C" int stp3_lift_splat_bwd(const stp3_lift_splat_desc* desc, const float* grad_out, const float* feat,
                                   const float* depth_logits, void* scratch, size_t scratch_bytes, float* grad_feat,
                                   float* grad_depth_logits, void* stream_) {
  LiftBwdParams p;
  if (const int rc = check_lift_splat_desc("stp3_lift_splat_bwd", desc, feat, depth_logits, kBwdMaxFrames, p.q)) return rc;
  STP3_CHECK_ARG(grad_out && scratch && grad_feat, "stp3_lift_splat_bwd: null pointer argument");
  STP3_CHECK_ARG(desc->feat_layout == 0, "stp3_lift_splat_bwd: feat must be NCHW (feat_layout 0)");
  return lift_splat_bwd_launch<false>("stp3_lift_splat_bwd", desc, grad_out, feat, depth_logits, scratch, scratch_bytes,
                                      grad_feat, grad_depth_logits, reinterpret_cast<cudaStream_t>(stream_), p);
}

extern "C" int stp3_lift_splat_bwd_cl(const stp3_lift_splat_desc* desc, const float* grad_out, const float* feat,
                                      const float* depth_logits, void* scratch, size_t scratch_bytes, float* grad_feat,
                                      float* grad_depth_logits, void* stream_) {
  LiftBwdParams p;
  if (const int rc = check_lift_splat_desc("stp3_lift_splat_bwd_cl", desc, feat, depth_logits, kBwdMaxFrames, p.q)) return rc;
  STP3_CHECK_ARG(grad_out && scratch && grad_feat, "stp3_lift_splat_bwd_cl: null pointer argument");
  STP3_CHECK_ARG(desc->feat_layout == 1, "stp3_lift_splat_bwd_cl: feat must be channels-last (feat_layout 1)");
  STP3_CHECK_ARG(desc->C % 2 == 0 && reinterpret_cast<uintptr_t>(feat) % 8 == 0 &&
                     reinterpret_cast<uintptr_t>(grad_feat) % 8 == 0,
                 "stp3_lift_splat_bwd_cl: C must be even and feat / grad_feat 8-byte aligned (float2 accesses)");
  return lift_splat_bwd_launch<true>("stp3_lift_splat_bwd_cl", desc, grad_out, feat, depth_logits, scratch,
                                     scratch_bytes, grad_feat, grad_depth_logits, reinterpret_cast<cudaStream_t>(stream_), p);
}
