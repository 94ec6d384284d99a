// ASPP branches + 1x1 projection as ONE back-to-back wgmma kernel (DeepLabHead of the temporal model,
// stp3/layers/convolutions.py:242-270: four conv/BN/ReLU branches of the same input, concatenated, then project.0).
//
// The unfused form writes the 4 x 128-channel concat tensor to HBM (4 x 246 MB for a 4-sample step) and reads it back
// (984 MB) -- the largest avoidable traffic of the dense path.  Here a CTA keeps an 8x16-pixel tile on chip:
//
//   for every branch b:   acc1  = sum_taps A(x, tap) . W_b[tap]            (wgmma, 64 rows per warpgroup, N = 128)
//                         P     = hi/lo split of relu(acc1 + bias_b)       (registers -> SHARED memory, written in the
//                                                                           128B-swizzled K-major operand layout)
//                         acc2 += P . W_proj[:, b-th 128 input channels]   (second MMA chain, A operand = P)
//   out = hi/lo split of relu(acc2 + per-image bias)                       (the global-pool branch is that bias)
//
// The same kernel runs the head's tail, 3x3 conv/BN/ReLU -> 1x1 classifier (convolutions.py:272-280), as a ONE-branch
// instance (9 taps, two input K blocks, classifier rows padded to 128, no ReLU on the output).
//
// Same precision scheme as conv_igemm.cu (bf16 hi/lo planes, hi*hi + hi*lo + lo*hi, fp32 accumulation), so the result
// matches the unfused path to the last few bits of the split.
//
//   warps : 0..7 = two warpgroups (rows 0..63 / 64..127 of the tile; each reads back only its own rows of P), 8 = TMA
//           producer (activation ring + weight ring)
//   smem  : 2 activation stages (64 KB) + 2 weight stages (64 KB) + P (2 K-blocks x hi/lo x 16 KB = 64 KB) = 192 KB
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kAsppThreads = 288;                 // 8 + 1 warps
constexpr int kAsppMaxBranches = 4;
constexpr int kAsppMaxTaps = 9 * kAsppMaxBranches;
constexpr int kAsppNA = 2, kAsppNB = 2;
constexpr int kAStage = 2 * 8 * 16 * 128;         // hi + lo planes of 8 image rows x 16 pixels x 64 channels
constexpr int kBStage = 2 * 128 * 128;            // hi + lo planes of the 128 weight rows
constexpr int kPPlane = 128 * 128;                // 128 pixel rows x 64 bf16
constexpr int kAsppHidden = 128;

struct AsppParams {
  int n_img, T, T_total, H, W;
  int tiles_x, tiles_y, n_tiles;
  int kblocks;
  int n_br;
  int br_tap0[kAsppMaxBranches + 1];
  signed char tap[kAsppMaxTaps][2];               // (dy, dx)
  const float* br_bias;                           // [n_br][128]
  const float* img_bias;                          // [n_img][128]
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int out_cstride, out_coff;
  int relu_out;                                   // ReLU on the projection output (ASPP: yes; conv3 -> classifier: no)
  int n_store;                                    // output channels stored (64 or 128): rows >= n_store of the projection are zero
};

__device__ __forceinline__ bool aspp_tap_is_padding(const AsppParams& p, int t, int oy_tile, int ox0) {
  const int ylo = oy_tile + p.tap[t][0], yhi = oy_tile + 7 + p.tap[t][0];
  const int xlo = ox0 + p.tap[t][1], xhi = ox0 + 15 + p.tap[t][1];
  return yhi < 0 || ylo >= p.H || xhi < 0 || xlo >= p.W;
}

__global__ void __launch_bounds__(kAsppThreads, 1)
aspp_fused_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_w, const AsppParams p) {
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* a_ring = smem;
  unsigned char* b_ring = a_ring + kAsppNA * kAStage;
  unsigned char* p_buf = b_ring + kAsppNB * kBStage;            // [kb2][hi | lo][128 rows x 128 B]
  float* s_bias = reinterpret_cast<float*>(p_buf + 4 * kPPlane);   // [n_br][128]
  float* s_wb = s_bias + kAsppMaxBranches * kAsppHidden;           // [2 warpgroups][128] per-image bias
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_wb + 2 * kAsppHidden);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kAsppNA;
  uint64_t* b_full = a_empty + kAsppNA;
  uint64_t* b_empty = b_full + kAsppNB;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    ptx::prefetch_tmap(&tm_a_hi); ptx::prefetch_tmap(&tm_a_lo); ptx::prefetch_tmap(&tm_w);
    for (int i = 0; i < kAsppNA; ++i) { ptx::mbar_init(&a_full[i], 1); ptx::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < kAsppNB; ++i) { ptx::mbar_init(&b_full[i], 1); ptx::mbar_init(&b_empty[i], 2); }
    ptx::fence_mbar_init();
  }
  for (int i = threadIdx.x; i < p.n_br * kAsppHidden; i += blockDim.x) s_bias[i] = p.br_bias[i];
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int proj_blk0 = p.br_tap0[p.n_br] * p.kblocks;          // first projection block of the weight tensor

  if (warp == 8) {
    // ===================== TMA producer =====================
    ptx::griddep_wait();
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    auto load_b = [&](int blk) {                   // weight block `blk`: [hi 128 rows][lo 128 rows]
      ptx::mbar_wait(&b_empty[bs], bph ^ 1);
      if (ptx::elect_one_sync()) {
        unsigned char* dst = b_ring + (size_t)bs * kBStage;
        ptx::mbar_arrive_expect_tx(&b_full[bs], (uint32_t)kBStage);
        ptx::tma_load_2d(dst, &tm_w, &b_full[bs], 0, blk * 256);
        ptx::tma_load_2d(dst + 128 * 128, &tm_w, &b_full[bs], 0, blk * 256 + 128);
      }
      __syncwarp();
      if (++bs == kAsppNB) { bs = 0; bph ^= 1; }
    };
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      const int bidx = img / p.T, tidx = img % p.T;
      for (int s = 0; s < p.n_br; ++s) {
        for (int t = p.br_tap0[s]; t < p.br_tap0[s + 1]; ++t) {
          if (aspp_tap_is_padding(p, t, oy_tile, ox0)) continue;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            ptx::mbar_wait(&a_empty[as], aph ^ 1);
            if (ptx::elect_one_sync()) {
              unsigned char* sa = a_ring + (size_t)as * kAStage;
              ptx::mbar_arrive_expect_tx(&a_full[as], (uint32_t)kAStage);
              ptx::tma_load_5d(sa, &tm_a_hi, &a_full[as], kb * 64, ox0 + p.tap[t][1], oy_tile + p.tap[t][0], tidx, bidx);
              ptx::tma_load_5d(sa + kAStage / 2, &tm_a_lo, &a_full[as], kb * 64, ox0 + p.tap[t][1], oy_tile + p.tap[t][0], tidx, bidx);
            }
            __syncwarp();
            if (++as == kAsppNA) { as = 0; aph ^= 1; }
            load_b(t * p.kblocks + kb);
          }
        }
        load_b(proj_blk0 + s * 2); load_b(proj_blk0 + s * 2 + 1);   // projection weights of this branch
      }
    }
  } else {
    // ===================== two warpgroups: branch MMAs, conversion to P, projection, output =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int wtid = threadIdx.x & 127;
    const bool wg_leader = wtid == 0;
    const int row0 = wg * 64 + wq * 16 + (lane >> 2);       // accumulator rows of this thread: row0, row0 + 8
    const int cq = 2 * (lane & 3);                           // first of its two columns in every 8-column group
    float* wb = s_wb + wg * kAsppHidden;
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    int pend_a = -1, pend_b = -1;               // ring slots read by the last committed wgmma group
    auto release = [&]() {
      if (wg_leader) {
        if (pend_a >= 0) ptx::mbar_arrive(&a_empty[pend_a]);
        if (pend_b >= 0) ptx::mbar_arrive(&b_empty[pend_b]);
      }
      pend_a = pend_b = -1;
    };
    auto issue = [&](float* acc, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, uint32_t accumulate,
                     int slot_a, int slot_b) {
      const uint64_t da_hi = wg::desc_k_sw128(a_hi), da_lo = wg::desc_k_sw128(a_lo);
      const uint64_t db_hi = wg::desc_k_sw128(b_hi), db_lo = wg::desc_k_sw128(b_lo);
      wg::fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t koff = (uint64_t)((k * 32) >> 4);
        wg::mma_bf16<kAsppHidden>(acc, da_hi + koff, db_hi + koff, accumulate | (uint32_t)k);
        wg::mma_bf16<kAsppHidden>(acc, da_hi + koff, db_lo + koff, 1);
        wg::mma_bf16<kAsppHidden>(acc, da_lo + koff, db_hi + koff, 1);
      }
      wg::commit();
      wg::wait<1>();
      release();
      pend_a = slot_a; pend_b = slot_b;
    };
    ptx::griddep_wait();
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      ptx::bar_sync(1 + wg, 128);                // the previous tile's output has read the per-image bias
      // written by the preceding (PDL-overlapped) pool_bias kernel: coherent loads
      wb[wtid] = *(reinterpret_cast<const volatile float*>(p.img_bias) + (size_t)img * kAsppHidden + wtid);
      float acc2[kAsppHidden / 2];
      for (int s = 0; s < p.n_br; ++s) {
        // ---- main(s): acc1 = sum over the branch's taps
        float acc1[kAsppHidden / 2];
        uint32_t accumulate = 0;
        for (int t = p.br_tap0[s]; t < p.br_tap0[s + 1]; ++t) {
          if (aspp_tap_is_padding(p, t, oy_tile, ox0)) continue;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            ptx::mbar_wait(&a_full[as], aph);
            ptx::mbar_wait(&b_full[bs], bph);
            const uint32_t a_hi = ptx::smem_u32(a_ring + (size_t)as * kAStage) + (uint32_t)(wg * 64 * 128);
            const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)bs * kBStage);
            issue(acc1, a_hi, a_hi + kAStage / 2, b_hi, b_hi + 128 * 128, accumulate, as, bs);
            accumulate = 1;
            if (++as == kAsppNA) { as = 0; aph ^= 1; }
            if (++bs == kAsppNB) { bs = 0; bph ^= 1; }
          }
        }
        wg::wait<0>();                             // also: the previous branch's projection has read P
        release();
        // ---- P = hi/lo split of relu(acc1 + bias): column c -> K block c / 64, 16-byte chunk (c % 64) / 8 of the
        // 128-byte row, XOR-swizzled with the row index (the layout TMA writes for a SWIZZLE_128B K-major operand)
        const float* bias = s_bias + s * kAsppHidden;
#pragma unroll
        for (int g8 = 0; g8 < 16; ++g8) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row0 + 8 * h;
            const float x0 = fmaxf(acc1[4 * g8 + 2 * h] + bias[8 * g8 + cq], 0.f);
            const float x1 = fmaxf(acc1[4 * g8 + 2 * h + 1] + bias[8 * g8 + cq + 1], 0.f);
            const uint32_t hw = ptx::pack_bf16x2(x0, x1);
            const uint32_t lw = ptx::pack_bf16x2(x0 - __uint_as_float(hw << 16), x1 - __uint_as_float(hw & 0xFFFF0000u));
            unsigned char* dst = p_buf + (size_t)(g8 >> 3) * 2 * kPPlane + (size_t)row * 128 +
                                 ((((uint32_t)g8 & 7u) ^ (uint32_t)(row & 7)) << 4) + cq * 2;
            *reinterpret_cast<uint32_t*>(dst) = hw;
            *reinterpret_cast<uint32_t*>(dst + kPPlane) = lw;
          }
        }
        ptx::fence_proxy_async();                  // the generic-proxy stores above are read by the tensor core (async proxy)
        ptx::bar_sync(1 + wg, 128);
        // ---- proj(s): acc2 (+)= P . W_proj[:, branch s]
        for (int kb2 = 0; kb2 < 2; ++kb2) {
          ptx::mbar_wait(&b_full[bs], bph);
          const uint32_t a_hi = ptx::smem_u32(p_buf + (size_t)kb2 * 2 * kPPlane) + (uint32_t)(wg * 64 * 128);
          const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)bs * kBStage);
          issue(acc2, a_hi, a_hi + kPPlane, b_hi, b_hi + 128 * 128, (s > 0 || kb2 > 0) ? 1u : 0u, -1, bs);
          if (++bs == kAsppNB) { bs = 0; bph ^= 1; }
        }
      }
      wg::wait<0>();
      release();
      // ---- output of the projection: relu(acc2 + per-image bias) -> hi/lo planes
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        const int oy = oy_tile + (row >> 4), ox = ox0 + (row & 15);
        if (oy >= p.H || ox >= p.W) continue;
        const size_t pix = ((size_t)img * p.H + oy) * p.W + ox;
#pragma unroll
        for (int g8 = 0; g8 < 16; ++g8) {
          const int c = 8 * g8 + cq;
          if (c >= p.n_store) continue;
          float x0 = acc2[4 * g8 + 2 * h] + wb[c];
          float x1 = acc2[4 * g8 + 2 * h + 1] + wb[c + 1];
          if (p.relu_out) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          const uint32_t hw = ptx::pack_bf16x2(x0, x1);
          const uint32_t lw = ptx::pack_bf16x2(x0 - __uint_as_float(hw << 16), x1 - __uint_as_float(hw & 0xFFFF0000u));
          const size_t off = pix * p.out_cstride + p.out_coff + c;
          *reinterpret_cast<uint32_t*>(p.out_hi + off) = hw;
          *reinterpret_cast<uint32_t*>(p.out_lo + off) = lw;
        }
      }
    }
  }
}

typedef CUresult (*PFN_tmapEncodeTiledA)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                         CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_tmapEncodeTiledA aspp_encode_fn() {
  static PFN_tmapEncodeTiledA fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiledA>(ptr);
  }
  return fn;
}

}  // namespace stp3

using namespace stp3;

extern "C" int stp3_aspp_fused_fwd(const stp3_aspp_desc* d, const void* x_hi, const void* x_lo, const void* w,
                                   const float* br_bias, const float* img_bias, void* y_hi, void* y_lo, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STP3_CHECK_ARG(d && x_hi && x_lo && w && br_bias && img_bias && y_hi && y_lo, "stp3_aspp_fused_fwd: null pointer argument");
  STP3_CHECK_ARG(d->B > 0 && d->T > 0 && d->H > 0 && d->W > 0, "non-positive dimension");
  STP3_CHECK_ARG(d->in_cstride % 64 == 0 && d->cin % 64 == 0 && d->cin > 0 && d->cin <= d->in_cstride, "input channels: multiples of 64");
  STP3_CHECK_ARG(d->n_br >= 1 && d->n_br <= kAsppMaxBranches, "1 .. 4 branches");
  const int n_store = d->n_store > 0 ? d->n_store : kAsppHidden;
  STP3_CHECK_ARG(n_store == 64 || n_store == 128, "n_store must be 64 or 128");
  STP3_CHECK_ARG(d->out_cstride % 16 == 0 && d->out_coff % 16 == 0 && d->out_coff + n_store <= d->out_cstride &&
                 (reinterpret_cast<uintptr_t>(y_hi) & 31) == 0 && (reinterpret_cast<uintptr_t>(y_lo) & 31) == 0,
                 "output planes: n_store channels at a 16-channel aligned offset, 32-byte aligned");
  PFN_tmapEncodeTiledA enc = aspp_encode_fn();
  if (!enc) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
  AsppParams p;
  p.n_img = d->B * d->T; p.T = d->T; p.T_total = d->T; p.H = d->H; p.W = d->W;
  p.tiles_x = ceil_div(d->W, 16); p.tiles_y = ceil_div(d->H, 8);
  const long long nt = (long long)p.n_img * p.tiles_x * p.tiles_y;
  STP3_CHECK_ARG(nt < (1ll << 31), "grid too large");
  p.n_tiles = (int)nt;
  p.kblocks = d->cin / 64; p.n_br = d->n_br;
  int t = 0;
  for (int b = 0; b < d->n_br; ++b) {
    STP3_CHECK_ARG(d->n_taps[b] >= 1 && d->n_taps[b] <= 9, "1 .. 9 taps per branch");
    p.br_tap0[b] = t;
    bool centre = false;
    for (int i = 0; i < d->n_taps[b]; ++i, ++t) {
      p.tap[t][0] = d->taps[b][i][0]; p.tap[t][1] = d->taps[b][i][1];
      centre |= d->taps[b][i][0] == 0 && d->taps[b][i][1] == 0;
    }
    STP3_CHECK_ARG(centre, "every branch needs its centre tap (padding skips rely on it)");
  }
  for (int b = d->n_br; b <= kAsppMaxBranches; ++b) p.br_tap0[b] = t;
  p.br_bias = br_bias; p.img_bias = img_bias;
  p.out_hi = static_cast<__nv_bfloat16*>(y_hi); p.out_lo = static_cast<__nv_bfloat16*>(y_lo);
  p.out_cstride = d->out_cstride; p.out_coff = d->out_coff;
  p.relu_out = d->no_relu ? 0 : 1; p.n_store = n_store;

  CUtensorMap tm_hi, tm_lo, tm_w;
  {
    const cuuint64_t dims[5] = {(cuuint64_t)d->in_cstride, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->T, (cuuint64_t)d->B};
    const cuuint64_t strides[4] = {(cuuint64_t)d->in_cstride * 2, (cuuint64_t)d->W * d->in_cstride * 2,
                                   (cuuint64_t)d->H * d->W * d->in_cstride * 2, (cuuint64_t)d->T * d->H * d->W * d->in_cstride * 2};
    const cuuint32_t box[5] = {64, 16, 8, 1, 1};
    const cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r1 = enc(&tm_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x_hi), dims, strides, box, es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CUresult r2 = enc(&tm_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x_lo), dims, strides, box, es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
      return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation) failed: %d %d", (int)r1, (int)r2);
    const int n_blocks = t * p.kblocks + 2 * d->n_br;
    const cuuint64_t wd[2] = {64, (cuuint64_t)n_blocks * 256};
    const cuuint64_t ws[1] = {128};
    const cuuint32_t wb[2] = {64, 128};
    const cuuint32_t we[2] = {1, 1};
    CUresult r3 = enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), wd, ws, wb, we,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r3 != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r3);
  }
  const size_t smem_bytes = 1024 + (size_t)kAsppNA * kAStage + (size_t)kAsppNB * kBStage + 4 * (size_t)kPPlane +
                            (kAsppMaxBranches + 2) * kAsppHidden * sizeof(float) + 2 * (kAsppNA + kAsppNB) * 8;
  static thread_local int attr_dev = -1;           // once per device: the attribute call costs microseconds per eager launch
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  if (attr_dev != cur_dev) {
    STP3_CUDA_OK(cudaFuncSetAttribute(aspp_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr_dev = cur_dev;
  }
  int num_sms = 132;
  cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, cur_dev);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(nt < num_sms ? nt : num_sms)); cfg.blockDim = dim3(kAsppThreads);
  cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = stp3_pdl_enabled("STP3_FUSED_PDL") ? 1 : 0;
  // The kernel never executes griddepcontrol.launch_dependents: its dependents are released when the grid completes
  // (see block_fused.cu); it still starts early behind its predecessor.
  STP3_CUDA_OK(cudaLaunchKernelEx(&cfg, aspp_fused_kernel, tm_hi, tm_lo, tm_w, p));
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
