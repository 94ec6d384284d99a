// Tail of a TemporalBlock as ONE back-to-back wgmma kernel (stp3/layers/temporal.py:426-489):
//
//   path 0 = causal (2,3,3) conv/BN/ReLU of mid_0      path 1 = (1,3,3) conv/BN/ReLU of mid_1      path 2 = 1x1x1 conv/BN/ReLU of x
//   out    = relu(BN(aggregation 1x1x1 of [path 0 | path 1 | path 2 | pyramid pooling])) + (projection(x) | x)
//
// (mid_0 / mid_1 = the paths' 1x1x1 entry convolutions, produced by a preceding stp3_conv_fwd launch).  The unfused form
// writes the three paths into a 128-channel concat tensor and reads it back (2 x 246 MB per block and 4-sample step) and
// needs one more pass over x for path 2 / the projection.  Here a CTA keeps an 8x16-pixel tile on chip:
//
//   (taps of one kernel column share ONE activation load: the box holds 8 + 2 image rows, tap j reads it shifted by j rows)
//   main    : the path chains one after the other, each into a register accumulator (its own input tensor, tap list,
//             MMA width N and K-step range); chain c's columns are the hidden channels [tmem_col, tmem_col + N)
//   convert : straight from the registers: add the (per-image) bias, ReLU, split to bf16 hi/lo and write the 8-channel
//             pieces of the compacted 128-channel operand P into shared memory (128B-swizzled K-major)
//   proj    : acc2 = P . W_agg  (N = 64);  acc3 = x_tile . W_projection (N = 64) when the block changes its width
//   final   : out = relu(acc2 + per-image bias) + (acc3 + per-image bias | x), hi/lo planes, per-image column sums
//
// Two warpgroups own rows 0..63 / 64..127 of the tile (the A operand of P is a warpgroup's own rows, so P needs only a
// warpgroup barrier); warp 8 is the TMA producer.  Same precision scheme as conv_igemm.cu (bf16 hi/lo planes, three
// MMAs per product, fp32 accumulation).
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kBlkThreads = 288;                  // 2 warpgroups + the producer warp
constexpr int kBlkMaxChains = 3;
constexpr int kBlkMaxTaps = 32;                 // 18 + 9 + 1 path taps + the projection's
constexpr int kBlkNA = 2, kBlkNB = 4;          // 200 KB of operand rings and P in 227 KB of shared memory
constexpr int kBlkBoxRows = 10;                   // 8 image rows + 2: one activation load serves the three dy taps of a kernel column
constexpr int kBlkAStage = 2 * kBlkBoxRows * 16 * 128;
constexpr int kBlkMaxGroups = 16;
constexpr int kBlkBRows = 64;                     // weight rows per plane: chains are at most 64 wide
constexpr int kBlkBStage = 2 * kBlkBRows * 128;
constexpr int kBlkPPlane = 128 * 128;

struct BlkChain {
  int src;                  // 0 = mid tensor, 1 = x tensor
  int cin_off;              // first channel of the 64-channel K block read from the source
  int tap0, ntaps;
  int grp0, ngrp;           // tap groups: runs of <= 3 taps with the same (dt, dx) and consecutive dy share one activation load
  int n_mma;                // MMA width (multiple of 16)
  int tmem_col;             // first hidden column of the chain's outputs
  int ks_first, ks_end;     // K = 16 steps that carry data
  int wblk0;                // first weight block (one per tap)
};

struct BlkParams {
  int n_img, T, H, W;
  int tiles_x, tiles_y, n_tiles;
  int n_chain;
  BlkChain chain[kBlkMaxChains];
  int has_res_proj;         // acc3 = x . W_projection
  BlkChain res;
  signed char tap[kBlkMaxTaps][4];        // (dt, dy, dx)
  unsigned char gstart[kBlkMaxGroups], gsize[kBlkMaxGroups];   // first tap / number of taps of every group
  int piece_col[16];        // hidden column of the 8-channel piece pp of P, -1 = zeros
  const float* hid_bias;    // [n_img][128] bias of the hidden channels in P order
  const float* img_bias;    // [n_img][64]  aggregation bias (+ pyramid-pooling branch)
  const float* res_bias;    // [n_img][64]  projection bias (has_res_proj) or null
  const __nv_bfloat16* res_hi;            // identity residual (x planes) when !has_res_proj
  const __nv_bfloat16* res_lo;
  int res_cstride;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int out_cstride;
  float* sum_part;          // [gridDim.x * 8][n_img][64] or null
  int wagg_blk0;            // two weight blocks (K blocks of P) of the aggregation conv
};

// true if every input element the tap group touches for this 8x16 tile is zero padding
__device__ __forceinline__ bool blk_group_is_padding(const BlkParams& p, int g, int tidx, int oy_tile, int ox0) {
  const int t0 = p.gstart[g];
  const int tt = tidx + p.tap[t0][0];
  const int ylo = oy_tile + p.tap[t0][1], yhi = oy_tile + 7 + p.tap[t0][1] + p.gsize[g] - 1;
  const int xlo = ox0 + p.tap[t0][2], xhi = ox0 + 15 + p.tap[t0][2];
  return tt < 0 || tt >= p.T || yhi < 0 || ylo >= p.H || xhi < 0 || xlo >= p.W;
}

__global__ void __launch_bounds__(kBlkThreads, 1)
block_fused_kernel(const __grid_constant__ CUtensorMap tm_m_hi, const __grid_constant__ CUtensorMap tm_m_lo,
                   const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                   const __grid_constant__ CUtensorMap tm_w, const BlkParams p) {
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* a_ring = smem;
  unsigned char* b_ring = a_ring + kBlkNA * kBlkAStage;
  unsigned char* p_buf = b_ring + kBlkNB * kBlkBStage;          // [kb2][hi | lo][128 rows x 128 B]
  float* s_hb = reinterpret_cast<float*>(p_buf + 4 * kBlkPPlane);   // [2 warpgroups][128] hidden bias of the image
  float* s_wb = s_hb + 2 * 128;                                     // [2 warpgroups][128] img_bias (64) | res_bias (64)
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_wb + 2 * 128);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kBlkNA;
  uint64_t* b_full = a_empty + kBlkNA;
  uint64_t* b_empty = b_full + kBlkNB;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    ptx::prefetch_tmap(&tm_m_hi); ptx::prefetch_tmap(&tm_m_lo); ptx::prefetch_tmap(&tm_x_hi); ptx::prefetch_tmap(&tm_x_lo);
    ptx::prefetch_tmap(&tm_w);
    for (int i = 0; i < kBlkNA; ++i) { ptx::mbar_init(&a_full[i], 1); ptx::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < kBlkNB; ++i) { ptx::mbar_init(&b_full[i], 1); ptx::mbar_init(&b_empty[i], 2); }
    ptx::fence_mbar_init();
  }
  // P pieces without a hidden column stay zero for the kernel's lifetime
  for (int i = threadIdx.x; i < 4 * kBlkPPlane / 16; i += blockDim.x) reinterpret_cast<uint4*>(p_buf)[i] = make_uint4(0u, 0u, 0u, 0u);
  ptx::fence_proxy_async();
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  if (warp == 8) {
    // ===================== TMA producer =====================
    ptx::griddep_wait();
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    auto load_a = [&](int src, int c, int x, int y, int t, int b) {
      ptx::mbar_wait(&a_empty[as], aph ^ 1);
      if (ptx::elect_one_sync()) {
        unsigned char* sa = a_ring + (size_t)as * kBlkAStage;
        ptx::mbar_arrive_expect_tx(&a_full[as], (uint32_t)kBlkAStage);
        ptx::tma_load_5d(sa, src ? &tm_x_hi : &tm_m_hi, &a_full[as], c, x, y, t, b);
        ptx::tma_load_5d(sa + kBlkAStage / 2, src ? &tm_x_lo : &tm_m_lo, &a_full[as], c, x, y, t, b);
      }
      __syncwarp();
      if (++as == kBlkNA) { as = 0; aph ^= 1; }
    };
    // weight block `blk` = [hi 128 rows][lo 128 rows]; output column n of an N-wide chain is row n (n < N/2) or
    // 64 + n - N/2 of each plane; only those rows are fetched (boxes of 8 rows)
    auto load_b = [&](int blk, int n_mma) {
      ptx::mbar_wait(&b_empty[bs], bph ^ 1);
      if (ptx::elect_one_sync()) {
        unsigned char* dst = b_ring + (size_t)bs * kBlkBStage;
        const int rows = n_mma / 2;
        ptx::mbar_arrive_expect_tx(&b_full[bs], (uint32_t)(2 * n_mma * 128));
        for (int r8 = 0; r8 < rows; r8 += 8) {
          for (int h = 0; h < 2; ++h) {
            ptx::tma_load_2d(dst + (h * rows + r8) * 128, &tm_w, &b_full[bs], 0, blk * 256 + h * 64 + r8);
            ptx::tma_load_2d(dst + kBlkBRows * 128 + (h * rows + r8) * 128, &tm_w, &b_full[bs], 0, blk * 256 + 128 + h * 64 + r8);
          }
        }
      }
      __syncwarp();
      if (++bs == kBlkNB) { bs = 0; bph ^= 1; }
    };
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      const int bidx = img / p.T, tidx = img % p.T;
      for (int c = 0; c < p.n_chain; ++c) {
        const BlkChain& ch = p.chain[c];
        for (int g = ch.grp0; g < ch.grp0 + ch.ngrp; ++g) {
          if (blk_group_is_padding(p, g, tidx, oy_tile, ox0)) continue;
          const int t0 = p.gstart[g];
          load_a(ch.src, ch.cin_off, ox0 + p.tap[t0][2], oy_tile + p.tap[t0][1], tidx + p.tap[t0][0], bidx);
          for (int j = 0; j < p.gsize[g]; ++j) load_b(ch.wblk0 + (t0 + j - ch.tap0), ch.n_mma);
        }
      }
      load_b(p.wagg_blk0, 64); load_b(p.wagg_blk0 + 1, 64);
      if (p.has_res_proj) { load_a(1, p.res.cin_off, ox0, oy_tile, tidx, bidx); load_b(p.res.wblk0, 64); }
    }
  } else {
    // ===================== two warpgroups: MMA, convert, projection, output =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int wtid = threadIdx.x & 127;
    const bool wg_leader = wtid == 0;
    const int row0 = wg * 64 + wq * 16 + (lane >> 2);       // accumulator rows of this thread: row0, row0 + 8
    const int cq = 2 * (lane & 3);                           // first of its two columns in every 8-column group
    float* hb = s_hb + wg * 128;
    float* wb = s_wb + wg * 128;
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    int pend_a = -1, pend_b = -1;               // ring slots read by the last committed wgmma group
    auto release = [&]() {
      if (wg_leader) {
        if (pend_a >= 0) ptx::mbar_arrive(&a_empty[pend_a]);
        if (pend_b >= 0) ptx::mbar_arrive(&b_empty[pend_b]);
      }
      pend_a = pend_b = -1;
    };
    // acc (+)= A . B over k in [k0, k1) with hi*hi + hi*lo + lo*hi, then commit and release the previous group's slots
    auto issue = [&](float* acc, int n, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, int k0, int k1,
                     uint32_t accumulate, int slot_a, int slot_b) {
      const uint64_t da_hi = wg::desc_k_sw128(a_hi), da_lo = wg::desc_k_sw128(a_lo);
      const uint64_t db_hi = wg::desc_k_sw128(b_hi), db_lo = wg::desc_k_sw128(b_lo);
      wg::fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < k0 || k >= k1) continue;
        const uint64_t koff = (uint64_t)((k * 32) >> 4);
        wg::mma_bf16_n<64>(n, acc, da_hi + koff, db_hi + koff, accumulate | (uint32_t)(k > k0));
        wg::mma_bf16_n<64>(n, acc, da_hi + koff, db_lo + koff, 1);
        wg::mma_bf16_n<64>(n, acc, da_lo + koff, db_hi + koff, 1);
      }
      wg::commit();
      wg::wait<1>();
      release();
      pend_a = slot_a; pend_b = slot_b;
    };
    float sacc[16];                              // column sums of this thread's columns (8 groups of 2)
#pragma unroll
    for (int i = 0; i < 16; ++i) sacc[i] = 0.f;
    int sum_img = -1;
    auto flush_sums = [&](int img_) {            // per column: sum over the 8 row pairs of the warp, once per image
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float v = sacc[i];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (lane < 4) p.sum_part[(((size_t)blockIdx.x * 8 + warp) * p.n_img + img_) * 64 + 8 * (i >> 1) + cq + (i & 1)] = v;
        sacc[i] = 0.f;
      }
    };
    ptx::griddep_wait();
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      const int tidx = img % p.T;
      if (p.sum_part && img != sum_img) {        // tiles come in image order
        if (sum_img >= 0) flush_sums(sum_img);
        sum_img = img;
      }
      ptx::bar_sync(1 + wg, 128);                // the previous tile is done with this warpgroup's bias rows
      {                                          // bias rows of this image (written by a preceding small kernel)
        const volatile float* hsrc = p.hid_bias + (size_t)img * 128;
        hb[wtid] = hsrc[wtid];
        const volatile float* isrc = p.img_bias + (size_t)img * 64;
        if (wtid < 64) wb[wtid] = isrc[wtid];
        else if (p.res_bias) wb[wtid] = *(reinterpret_cast<const volatile float*>(p.res_bias) + (size_t)img * 64 + wtid - 64);
      }
      ptx::bar_sync(1 + wg, 128);
      // ---------- main: every chain into registers, converted into its pieces of P
      for (int c = 0; c < p.n_chain; ++c) {
        const BlkChain& ch = p.chain[c];
        float acc[32];
        uint32_t accumulate = 0;
        for (int g = ch.grp0; g < ch.grp0 + ch.ngrp; ++g) {
          if (blk_group_is_padding(p, g, tidx, oy_tile, ox0)) continue;
          ptx::mbar_wait(&a_full[as], aph);
          const uint32_t a_hi0 = ptx::smem_u32(a_ring + (size_t)as * kBlkAStage) + (uint32_t)(wg * 64 * 128);
          for (int j = 0; j < p.gsize[g]; ++j) {
            ptx::mbar_wait(&b_full[bs], bph);
            const uint32_t a_hi = a_hi0 + (uint32_t)(j * 16 * 128);          // tap j of the group: shifted by j image rows
            const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)bs * kBlkBStage);
            issue(acc, ch.n_mma, a_hi, a_hi + kBlkAStage / 2, b_hi, b_hi + kBlkBRows * 128, ch.ks_first, ch.ks_end,
                  accumulate, j + 1 == p.gsize[g] ? as : -1, bs);
            accumulate = 1;
            if (++bs == kBlkNB) { bs = 0; bph ^= 1; }
          }
          if (++as == kBlkNA) { as = 0; aph ^= 1; }
        }
        wg::wait<0>();
        release();
        // convert: piece pp of P holds hidden columns [piece_col[pp], +8) = 8-column group (piece_col - tmem_col) / 8
        for (int pp = 0; pp < 16; ++pp) {
          const int col = p.piece_col[pp] - ch.tmem_col;
          if (p.piece_col[pp] < 0 || col < 0 || col >= ch.n_mma) continue;
          const int grp8 = col >> 3;
#pragma unroll
          for (int g8 = 0; g8 < 8; ++g8) {               // chains are at most 64 wide: 8 groups of 8 columns
            if (g8 != grp8) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + 8 * h;
              const float x0 = fmaxf(acc[4 * g8 + 2 * h] + hb[pp * 8 + cq], 0.f);
              const float x1 = fmaxf(acc[4 * g8 + 2 * h + 1] + hb[pp * 8 + cq + 1], 0.f);
              const uint32_t hw = ptx::pack_bf16x2(x0, x1);
              const uint32_t lw = ptx::pack_bf16x2(x0 - __uint_as_float(hw << 16), x1 - __uint_as_float(hw & 0xFFFF0000u));
              unsigned char* dst = p_buf + (size_t)(pp >> 3) * 2 * kBlkPPlane + (size_t)row * 128 +
                                   ((((uint32_t)pp & 7u) ^ (uint32_t)(row & 7)) << 4) + cq * 2;
              *reinterpret_cast<uint32_t*>(dst) = hw;
              *reinterpret_cast<uint32_t*>(dst + kBlkPPlane) = lw;
            }
          }
        }
      }
      ptx::fence_proxy_async();                  // the generic-proxy stores above are read by the tensor core (async proxy)
      ptx::bar_sync(1 + wg, 128);
      // ---------- projection: acc2 = P . W_agg, acc3 = x . W_projection
      float acc2[32], acc3[32];
      for (int kb2 = 0; kb2 < 2; ++kb2) {
        ptx::mbar_wait(&b_full[bs], bph);
        const uint32_t a_hi = ptx::smem_u32(p_buf + (size_t)kb2 * 2 * kBlkPPlane) + (uint32_t)(wg * 64 * 128);
        const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)bs * kBlkBStage);
        issue(acc2, 64, a_hi, a_hi + kBlkPPlane, b_hi, b_hi + kBlkBRows * 128, 0, 4, kb2 > 0 ? 1u : 0u, -1, bs);
        if (++bs == kBlkNB) { bs = 0; bph ^= 1; }
      }
      if (p.has_res_proj) {
        ptx::mbar_wait(&a_full[as], aph);
        ptx::mbar_wait(&b_full[bs], bph);
        const uint32_t a_hi = ptx::smem_u32(a_ring + (size_t)as * kBlkAStage) + (uint32_t)(wg * 64 * 128);
        const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)bs * kBlkBStage);
        issue(acc3, 64, a_hi, a_hi + kBlkAStage / 2, b_hi, b_hi + kBlkBRows * 128, p.res.ks_first, p.res.ks_end, 0u, as, bs);
        if (++as == kBlkNA) { as = 0; aph ^= 1; }
        if (++bs == kBlkNB) { bs = 0; bph ^= 1; }
      }
      wg::wait<0>();
      release();
      // ---------- output: relu(acc2 + bias) + residual, two channels per 8-column group and row
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        const int oy = oy_tile + (row >> 4), ox = ox0 + (row & 15);
        if (oy >= p.H || ox >= p.W) continue;
        const size_t pix = ((size_t)img * p.H + oy) * p.W + ox;
#pragma unroll
        for (int g8 = 0; g8 < 8; ++g8) {
          const int c = 8 * g8 + cq;
          float v0 = fmaxf(acc2[4 * g8 + 2 * h] + wb[c], 0.f);
          float v1 = fmaxf(acc2[4 * g8 + 2 * h + 1] + wb[c + 1], 0.f);
          if (p.has_res_proj) {
            v0 += acc3[4 * g8 + 2 * h] + wb[64 + c];
            v1 += acc3[4 * g8 + 2 * h + 1] + wb[64 + c + 1];
          } else {                               // identity residual: the block's input planes
            const size_t off = pix * p.res_cstride + c;
            const uint32_t rh = *reinterpret_cast<const volatile uint32_t*>(p.res_hi + off);
            const uint32_t rl = *reinterpret_cast<const volatile uint32_t*>(p.res_lo + off);
            v0 += __uint_as_float(rh << 16) + __uint_as_float(rl << 16);
            v1 += __uint_as_float(rh & 0xFFFF0000u) + __uint_as_float(rl & 0xFFFF0000u);
          }
          const uint32_t hw = ptx::pack_bf16x2(v0, v1);
          const uint32_t lw = ptx::pack_bf16x2(v0 - __uint_as_float(hw << 16), v1 - __uint_as_float(hw & 0xFFFF0000u));
          const size_t off = pix * p.out_cstride + c;
          *reinterpret_cast<uint32_t*>(p.out_hi + off) = hw;
          *reinterpret_cast<uint32_t*>(p.out_lo + off) = lw;
          if (p.sum_part) { sacc[2 * g8] += v0; sacc[2 * g8 + 1] += v1; }
        }
      }
    }
    if (p.sum_part && sum_img >= 0) flush_sums(sum_img);
  }
}

typedef CUresult (*PFN_tmapEncodeTiledB)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                         CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_tmapEncodeTiledB blk_encode_fn() {
  static PFN_tmapEncodeTiledB fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiledB>(ptr);
  }
  return fn;
}

static int blk_num_sms() {
  static const int n = [] {
    int dev = 0, v = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();
  return n;
}

}  // namespace stp3

using namespace stp3;

extern "C" size_t stp3_block_fused_scratch_bytes(int n_img) {
  return (size_t)blk_num_sms() * 8 * (size_t)(n_img > 0 ? n_img : 0) * 64 * sizeof(float);
}

extern "C" int stp3_block_fused_fwd(const stp3_block_desc* d, const void* mid_hi, const void* mid_lo, const void* x_hi,
                                    const void* x_lo, const void* w, const float* hid_bias, const float* img_bias,
                                    const float* res_bias, void* y_hi, void* y_lo, float* col_sums, void* scratch,
                                    size_t scratch_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STP3_CHECK_ARG(d && mid_hi && mid_lo && x_hi && x_lo && w && hid_bias && img_bias && y_hi && y_lo,
                 "stp3_block_fused_fwd: null pointer argument");
  STP3_CHECK_ARG(d->B > 0 && d->T > 0 && d->H > 0 && d->W > 0, "non-positive dimension");
  STP3_CHECK_ARG(d->mid_cstride % 64 == 0 && d->x_cstride % 64 == 0 && d->out_cstride % 16 == 0 && d->out_cstride >= 64,
                 "channel strides: mid / x multiples of 64, out a multiple of 16 and >= 64");
  STP3_CHECK_ARG(d->n_chain >= 1 && d->n_chain <= kBlkMaxChains, "1 .. 3 path chains");
  STP3_CHECK_ARG((d->has_res_proj != 0) == (res_bias != nullptr), "res_bias is given exactly when the block has a projection");
  auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
  STP3_CHECK_ARG(al32(y_hi) && al32(y_lo) && al32(x_hi) && al32(x_lo), "planes must be 32-byte aligned");
  PFN_tmapEncodeTiledB enc = blk_encode_fn();
  if (!enc) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");

  BlkParams p;
  p.n_img = d->B * d->T; p.T = d->T; p.H = d->H; p.W = d->W;
  p.tiles_x = ceil_div(d->W, 16); p.tiles_y = ceil_div(d->H, 8);
  const long long nt = (long long)p.n_img * p.tiles_x * p.tiles_y;
  STP3_CHECK_ARG(nt < (1ll << 31), "grid too large");
  p.n_tiles = (int)nt;
  p.n_chain = d->n_chain;
  int t = 0, blk = 0, n_grp = 0;
  auto fill = [&](BlkChain& c, const stp3_block_chain& s) -> int {
    c.src = s.src; c.cin_off = s.cin_off; c.tap0 = t; c.ntaps = s.n_taps; c.n_mma = s.n_mma; c.tmem_col = s.tmem_col;
    c.ks_first = s.k_lo / 16; c.ks_end = s.k_hi / 16; c.wblk0 = blk;
    if (!(s.n_taps >= 1 && s.n_taps <= 18 && s.n_mma % 16 == 0 && s.n_mma >= 16 && s.n_mma <= 64 && s.tmem_col % 16 == 0 &&
          s.tmem_col + s.n_mma <= 144 && s.cin_off % 64 == 0 && s.k_lo % 16 == 0 && s.k_hi % 16 == 0 && s.k_lo < s.k_hi &&
          s.k_hi <= 64 && (s.src == 0 || s.src == 1)))
      return set_error(STP3_EINVAL, "stp3_block_fused_fwd: bad chain descriptor");
    bool centre = false;
    for (int i = 0; i < s.n_taps; ++i, ++t) {
      if (t >= kBlkMaxTaps) return set_error(STP3_EINVAL, "too many taps");
      p.tap[t][0] = s.taps[i][0]; p.tap[t][1] = s.taps[i][1]; p.tap[t][2] = s.taps[i][2]; p.tap[t][3] = 0;
      centre |= s.taps[i][0] == 0 && s.taps[i][1] == 0 && s.taps[i][2] == 0;
    }
    if (!centre) return set_error(STP3_EINVAL, "every chain needs its centre tap");
    // tap groups: consecutive taps with the same (dt, dx) and dy advancing by one
    c.grp0 = n_grp;
    for (int i = c.tap0; i < c.tap0 + c.ntaps;) {
      int g = 1;
      while (g < 3 && i + g < c.tap0 + c.ntaps && p.tap[i + g][0] == p.tap[i][0] && p.tap[i + g][2] == p.tap[i][2] &&
             p.tap[i + g][1] == p.tap[i][1] + g)
        ++g;
      if (n_grp >= kBlkMaxGroups) return set_error(STP3_EINVAL, "too many tap groups");
      p.gstart[n_grp] = (unsigned char)i; p.gsize[n_grp] = (unsigned char)g; ++n_grp;
      i += g;
    }
    c.ngrp = n_grp - c.grp0;
    blk += s.n_taps;
    return STP3_OK;
  };
  for (int c = 0; c < d->n_chain; ++c) { const int rc = fill(p.chain[c], d->chain[c]); if (rc) return rc; }
  p.wagg_blk0 = blk; blk += 2;
  p.has_res_proj = d->has_res_proj ? 1 : 0;
  if (p.has_res_proj) {
    STP3_CHECK_ARG(t < kBlkMaxTaps, "too many taps");
    stp3_block_chain rs = d->res;
    STP3_CHECK_ARG(rs.n_taps == 1 && rs.src == 1 && rs.n_mma == 64, "the projection chain is a 1x1 on x with 64 outputs");
    const int rc = fill(p.res, rs); if (rc) return rc;
  } else {
    p.res = p.chain[0];
  }
  for (int i = 0; i < 16; ++i) {
    STP3_CHECK_ARG(d->piece_col[i] < 0 || (d->piece_col[i] % 8 == 0 && d->piece_col[i] + 8 <= 144), "bad piece column");
    p.piece_col[i] = d->piece_col[i];
  }
  p.hid_bias = hid_bias; p.img_bias = img_bias; p.res_bias = res_bias;
  p.res_hi = static_cast<const __nv_bfloat16*>(x_hi); p.res_lo = static_cast<const __nv_bfloat16*>(x_lo);
  p.res_cstride = d->x_cstride;
  p.out_hi = static_cast<__nv_bfloat16*>(y_hi); p.out_lo = static_cast<__nv_bfloat16*>(y_lo); p.out_cstride = d->out_cstride;

  CUtensorMap tm[4], tm_w;
  const void* planes[4] = {mid_hi, mid_lo, x_hi, x_lo};
  for (int i = 0; i < 4; ++i) {
    const int cs = i < 2 ? d->mid_cstride : d->x_cstride;
    const cuuint64_t dims[5] = {(cuuint64_t)cs, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->T, (cuuint64_t)d->B};
    const cuuint64_t strides[4] = {(cuuint64_t)cs * 2, (cuuint64_t)d->W * cs * 2, (cuuint64_t)d->H * d->W * cs * 2,
                                   (cuuint64_t)d->T * d->H * d->W * cs * 2};
    const cuuint32_t box[5] = {64, 16, (cuuint32_t)kBlkBoxRows, 1, 1};
    const cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(&tm[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(planes[i]), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation %d) failed: %d", i, (int)r);
  }
  {
    const cuuint64_t wd[2] = {64, (cuuint64_t)blk * 256};
    const cuuint64_t ws[1] = {128};
    const cuuint32_t wb[2] = {64, 8};
    const cuuint32_t we[2] = {1, 1};
    CUresult r = enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), wd, ws, wb, we,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  }
  const size_t smem_bytes = 1024 + (size_t)kBlkNA * kBlkAStage + (size_t)kBlkNB * kBlkBStage + 4 * (size_t)kBlkPPlane +
                            4 * 128 * sizeof(float) + 2 * (kBlkNA + kBlkNB) * 8;
  static thread_local int attr_dev = -1;           // once per device: the attribute call costs microseconds per eager launch
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  if (attr_dev != cur_dev) {
    STP3_CUDA_OK(cudaFuncSetAttribute(block_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    attr_dev = cur_dev;
  }
  const int num_sms = blk_num_sms();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(nt < num_sms ? nt : num_sms)); cfg.blockDim = dim3(kBlkThreads);
  cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = stp3_pdl_enabled("STP3_FUSED_PDL") ? 1 : 0;
  p.sum_part = nullptr;
  if (col_sums) {
    const size_t need = (size_t)cfg.gridDim.x * 8 * p.n_img * 64 * sizeof(float);
    STP3_CHECK_ARG(scratch && scratch_bytes >= need, "col_sums: scratch missing or smaller than stp3_block_fused_scratch_bytes()");
    p.sum_part = static_cast<float*>(scratch);
    STP3_CUDA_OK(cudaMemsetAsync(p.sum_part, 0, need, stream));
  }
  // The back-to-back kernels never execute griddepcontrol.launch_dependents, so their dependents start only when the
  // grid has completed.  Each of them needs a whole SM; an early trigger would let a chain block_fused -> col_sum_reduce
  // -> pool_bias -> aspp_fused be resident at once, and such a chain was seen to stop making progress.  The kernel itself
  // still starts early behind its predecessor (griddepcontrol.wait before it reads what that predecessor wrote).
  STP3_CUDA_OK(cudaLaunchKernelEx(&cfg, block_fused_kernel, tm[0], tm[1], tm[2], tm[3], tm_w, p));
  STP3_CUDA_OK(cudaGetLastError());
  if (col_sums) return launch_col_sum_reduce(p.sum_part, (int)cfg.gridDim.x * 8, p.n_img, col_sums, stream);
  return STP3_OK;
}
