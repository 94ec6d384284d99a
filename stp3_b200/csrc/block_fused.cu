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
//   convert : straight from the registers: add the (per-image) bias, ReLU and split to bf16 hi/lo.  The packed fp32
//             accumulator fragment of two 8-column groups is the wgmma A fragment of 16 channels of the compacted
//             128-channel operand P, so P never leaves the registers
//   agg     : acc2 += P_k . W_agg[k] (register-A wgmma, N = 64) for every K = 16 step of P as soon as both of its
//             8-channel pieces exist; a step that straddles two chains keeps the first chain's half until the next one
//             completes it.  The steps are issued in increasing k, so acc2 sums exactly as the shared-memory P did
//   proj    : acc3 = x_tile . W_projection (N = 64) when the block changes its width, on the activation stage that
//             path 2 (the 1x1x1 chain of x, always the last chain) has loaded
//   final   : out = relu(acc2 + per-image bias) + (acc3 + per-image bias | x), hi/lo planes, per-image column sums
//   store   : the output tile is staged in path 2's activation stage, laid out as the TMA load wrote it (per plane
//             [pixel row][128 B], 128-byte swizzle), and leaves by one cp.async.bulk.tensor store per warpgroup and
//             plane; the identity residual x is read from the same bytes just before they are overwritten.  That
//             stage goes back to the producer once the stores have read it, early in the next tile, whose first
//             chains load into the other two stages
//
// Two warpgroups own rows 0..63 / 64..127 of the tile; warp 8 is the TMA producer, and its warpgroup hands its registers
// to the MMA warpgroups (setmaxnreg 40 / 232: a chain accumulator, acc2, acc3 and the P fragments live at once do not
// fit the 168 registers per thread of an even split, and ptxas would serialise the wgmma).  Same precision scheme as
// conv_igemm.cu (bf16 hi/lo planes, three MMAs per product, fp32 accumulation).  Every chain's MMA width, K-step count
// and place in P select compile-time issue sequences once per chain, so no wgmma sits behind a run-time width or
// K-skip branch.
//
//   smem : 3 activation stages (120 KB) + 4 weight stages (64 KB) + the aggregation weights, resident for the kernel's
//          lifetime (32 KB; they are the same for every tile)
#include <cuda_bf16.h>

#include "common.cuh"
#include "pipeline.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kBlkThreads = 384;                  // 2 MMA warpgroups + the producer warpgroup
constexpr int kBlkMaxChains = 3;
constexpr int kBlkMaxTaps = 32;                 // 18 + 9 + 1 path taps + the projection's
constexpr int kBlkNA = 3, kBlkNB = 4;
constexpr int kBlkBoxRows = 10;                   // 8 image rows + 2: one activation load serves the three dy taps of a kernel column
constexpr int kBlkAStage = 2 * kBlkBoxRows * 16 * 128;
constexpr int kBlkMaxGroups = 16;
constexpr int kBlkBRows = 64;                     // weight rows per plane: chains are at most 64 wide
constexpr int kBlkBStage = 2 * kBlkBRows * 128;
// the output tile is staged in path 2's activation stage: per plane its first 128 pixel rows of 128 bytes (64 channels),
// 1024-byte aligned for the 128-byte swizzle; each warpgroup stores its 64 rows as one box of 16 x kBlkStoreRows pixels
constexpr int kBlkStoreRows = 4;
static_assert(kBlkAStage / 2 >= 8 * 16 * 128 && (kBlkAStage / 2) % 1024 == 0, "an activation plane stages 128 pixels x 64 channels");
static_assert(16 * kBlkStoreRows == 64, "one store box per warpgroup: its 64 accumulator rows");

// shared memory, from the 1024-byte aligned base (the kernel carves it, the host sizes the launch from `bytes`)
struct BlkSmem {
  static constexpr int a_ring = 0;                                // kBlkNA activation stages
  static constexpr int b_ring = a_ring + kBlkNA * kBlkAStage;     // kBlkNB weight stages
  static constexpr int w_agg = b_ring + kBlkNB * kBlkBStage;      // the two aggregation blocks, as two weight stages
  static constexpr int hb = w_agg + 2 * kBlkBStage;               // fp32 [2 warpgroups][128] hidden bias of the image
  static constexpr int wb = hb + 2 * 128 * 4;                     // fp32 [2 warpgroups][128] img_bias (64) | res_bias (64)
  static constexpr int bars = wb + 2 * 128 * 4;                   // full / empty barriers of both rings, w_agg_full
  static constexpr size_t bytes = 1024 + bars + (2 * (kBlkNA + kBlkNB) + 1) * 8;   // + the alignment slack
};

// The two chain layouts the kernel is compiled for, i.e. the two TemporalBlock packs.  Per chain: MMA width N, the
// 8-channel pieces of P it produces (its column groups 0 .. npc - 1), the first of them:
//   kBlkThreePaths: three 33..40-channel paths at N = 48, pieces 0-4 | 5-9 | 10-14 (piece 15 is zero)
//   kBlkDiagPair  : the block-diagonal chain of both mid paths at N = 64, pieces 0-7, then path 2 at N = 32, pieces 8-11
// Chain 0 of the first layout ends in the middle of a K = 16 step of P; chain 1 completes that step.  Chain 2 issues its
// last half step with a zero second half.  K steps with no piece at all (the second layout's steps 6 and 7) are not
// issued: they would add exact zeros to acc2.
enum BlkLayout { kBlkThreePaths = 0, kBlkDiagPair = 1 };

struct BlkChain {
  int src;                  // 0 = mid tensor, 1 = x tensor
  int cin_off;              // first channel of the 64-channel K block read from the source
  int tap0, ntaps;
  int grp0, ngrp;           // tap groups: runs of <= 3 taps with the same (dt, dx) and consecutive dy share one activation load
  int n_mma;                // MMA width (multiple of 16)
  int tmem_col;             // first hidden column of the chain's outputs
  int ks_first, ks_end;     // K = 16 steps that carry data
  int wblk0;                // first weight block (one per tap)
  int pc0;                  // first 8-channel piece of P this chain produces
};

struct BlkParams {
  int n_img, T, H, W;
  int tiles_x, tiles_y, n_tiles;
  int n_chain;
  BlkChain chain[kBlkMaxChains];
  int has_res_proj;         // acc3 = x . W_projection, on the last chain's activation stage
  BlkChain res;
  signed char tap[kBlkMaxTaps][4];        // (dt, dy, dx)
  unsigned char gstart[kBlkMaxGroups], gsize[kBlkMaxGroups];   // first tap / number of taps of every group
  const float* hid_bias;    // [n_img][128] bias of the hidden channels in P order
  const float* img_bias;    // [n_img][64]  aggregation bias (+ pyramid-pooling branch)
  const float* res_bias;    // [n_img][64]  projection bias (has_res_proj) or null
  float* sum_part;          // [gridDim.x * 8][n_img][64] or null
  int wagg_blk0;            // two weight blocks (K blocks of P) of the aggregation conv
};

template <int V>
struct BlkC { static constexpr int value = V; };

// true if every input element the tap group touches for this 8x16 tile is zero padding
__device__ __forceinline__ bool blk_group_is_padding(const BlkParams& p, int g, int tidx, int oy_tile, int ox0) {
  const int t0 = p.gstart[g];
  const int tt = tidx + p.tap[t0][0];
  const int ylo = oy_tile + p.tap[t0][1], yhi = oy_tile + 7 + p.tap[t0][1] + p.gsize[g] - 1;
  const int xlo = ox0 + p.tap[t0][2], xhi = ox0 + 15 + p.tap[t0][2];
  return tt < 0 || tt >= p.T || yhi < 0 || ylo >= p.H || xhi < 0 || xlo >= p.W;
}

template <int LAYOUT>
__global__ void __launch_bounds__(kBlkThreads, 1)
block_fused_kernel(const __grid_constant__ CUtensorMap tm_m_hi, const __grid_constant__ CUtensorMap tm_m_lo,
                   const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                   const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_o_hi,
                   const __grid_constant__ CUtensorMap tm_o_lo, const BlkParams p) {
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* a_ring = smem + BlkSmem::a_ring;
  unsigned char* b_ring = smem + BlkSmem::b_ring;
  unsigned char* w_agg = smem + BlkSmem::w_agg;
  float* s_hb = reinterpret_cast<float*>(smem + BlkSmem::hb);
  float* s_wb = reinterpret_cast<float*>(smem + BlkSmem::wb);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BlkSmem::bars);
  Ring ra{bars, bars + kBlkNA, kBlkNA};
  Ring rb{bars + 2 * kBlkNA, bars + 2 * kBlkNA + kBlkNB, kBlkNB};
  uint64_t* w_agg_full = bars + 2 * (kBlkNA + kBlkNB);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    ptx::prefetch_tmap(&tm_m_hi); ptx::prefetch_tmap(&tm_m_lo); ptx::prefetch_tmap(&tm_x_hi); ptx::prefetch_tmap(&tm_x_lo);
    ptx::prefetch_tmap(&tm_w); ptx::prefetch_tmap(&tm_o_hi); ptx::prefetch_tmap(&tm_o_lo);
    ra.init(2); rb.init(2);
    ptx::mbar_init(w_agg_full, 2);               // one arrive.expect_tx per aggregation block
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  if (warp >= 8) {
    ptx::setmaxnreg_dec<40>();
    if (warp != 8) return;
    // ===================== TMA producer =====================
    // weight block `blk` = [hi 128 rows][lo 128 rows]; output column n of an N-wide chain is row n (n < N/2) or
    // 64 + n - N/2 of each plane; only those rows are fetched (boxes of 8 rows)
    auto fetch_b = [&](unsigned char* dst, uint64_t* bar, int blk, int n_mma) {
      const int rows = n_mma / 2;
      for (int r8 = 0; r8 < rows; r8 += 8) {
        for (int h = 0; h < 2; ++h) {
          ptx::tma_load_2d(dst + (h * rows + r8) * 128, &tm_w, bar, 0, blk * 256 + h * 64 + r8);
          ptx::tma_load_2d(dst + kBlkBRows * 128 + (h * rows + r8) * 128, &tm_w, bar, 0, blk * 256 + 128 + h * 64 + r8);
        }
      }
    };
    // module weights, not written by the predecessor: fetched before the dependency wait
    if (ptx::elect_one_sync()) {
      ptx::mbar_arrive_expect_tx(w_agg_full, 2 * 64 * 128);
      fetch_b(w_agg, w_agg_full, p.wagg_blk0, 64);
      ptx::mbar_arrive_expect_tx(w_agg_full, 2 * 64 * 128);
      fetch_b(w_agg + kBlkBStage, w_agg_full, p.wagg_blk0 + 1, 64);
    }
    __syncwarp();
    ptx::griddep_wait();
    auto load_a = [&](int src, int c, int x, int y, int t, int b) {
      ra.produce(kBlkAStage, [&](int s, uint64_t* bar) {
        unsigned char* sa = a_ring + (size_t)s * kBlkAStage;
        ptx::tma_load_5d(sa, src ? &tm_x_hi : &tm_m_hi, bar, c, x, y, t, b);
        ptx::tma_load_5d(sa + kBlkAStage / 2, src ? &tm_x_lo : &tm_m_lo, bar, c, x, y, t, b);
      });
    };
    auto load_b = [&](int blk, int n_mma) {
      rb.produce(2 * n_mma * 128, [&](int s, uint64_t* bar) { fetch_b(b_ring + (size_t)s * kBlkBStage, bar, blk, n_mma); });
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
      if (p.has_res_proj) load_b(p.res.wblk0, 64);          // its activations: the last chain's stage
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // ===================== two warpgroups: chains, conversion to P, aggregation, projection, output =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int wtid = threadIdx.x & 127;
    const int row0 = wg * 64 + wq * 16 + (lane >> 2);       // accumulator rows of this thread: row0, row0 + 8
    const int cq = 2 * (lane & 3);                           // first of its two columns in every 8-column group
    float* hb = s_hb + wg * 128;
    float* wb = s_wb + wg * 128;
    const uint32_t w_agg_u32 = ptx::smem_u32(w_agg);
    PendingSlots pend{ra.empty, rb.empty, wtid == 0};
    int out_slot = -1;                           // activation stage holding the previous tile's output until stored
    // acc (+)= A . B over KS K steps from k0 with hi*hi + hi*lo + lo*hi, then commit and release the previous group's slots
    auto issue = [&](auto n_c, auto ks_c, float* acc, uint32_t a_hi, uint32_t b_hi, int k0, uint32_t accumulate,
                     int slot_a, int slot_b) {
      constexpr int N = decltype(n_c)::value, KS = decltype(ks_c)::value;
      const uint64_t da_hi = wg::desc_k_sw128(a_hi) + (uint64_t)(2 * k0), da_lo = wg::desc_k_sw128(a_hi + kBlkAStage / 2) + (uint64_t)(2 * k0);
      const uint64_t db_hi = wg::desc_k_sw128(b_hi) + (uint64_t)(2 * k0), db_lo = wg::desc_k_sw128(b_hi + kBlkBRows * 128) + (uint64_t)(2 * k0);
      wg::fence();
#pragma unroll
      for (int k = 0; k < KS; ++k)
        wg::mma_hilo<N>(acc, da_hi + 2 * k, da_lo + 2 * k, db_hi + 2 * k, db_lo + 2 * k, k == 0 ? accumulate : 1u);
      wg::commit();
      wg::wait<1>();
      pend.release_and_defer(slot_a, slot_b);
    };
    // one K = 16 step of the aggregation: acc2 (+)= P_s . W_agg[s], P_s from registers (hi / lo A fragments)
    float acc2[32], acc3[32];
    auto agg_step = [&](int s, const uint32_t* f_hi, const uint32_t* f_lo) {
      const uint32_t b_hi = w_agg_u32 + (uint32_t)((s >> 2) * kBlkBStage);
      const uint64_t koff = (uint64_t)(2 * (s & 3));
      const uint64_t db_hi = wg::desc_k_sw128(b_hi) + koff, db_lo = wg::desc_k_sw128(b_hi + kBlkBRows * 128) + koff;
      wg::mma_hilo_rs<64>(acc2, f_hi, f_lo, db_hi, db_lo, s > 0 ? 1u : 0u);
    };
    uint32_t carry_hi[2] = {0u, 0u}, carry_lo[2] = {0u, 0u};   // the first half of a K step that straddles two chains
    int agg_next = 0;                           // next K step of the aggregation

    // one chain of one tile: its taps (and the projection on the same activation stage), then its pieces of P into acc2.
    // The first chain hands the previous tile's output stage back to the producer once its stores have read it (after
    // an issue, so the new group runs meanwhile).  The last chain (path 2, one group) keeps its activation stage as this
    // tile's output staging area: `stage`
    int stage = -1;
    auto run_chain = [&](auto first_c, auto n_c, auto npc_c, auto odd_c, auto close_c, const BlkChain& ch, int tidx,
                         int oy_tile, int ox0, bool with_proj, bool last_chain) {
      constexpr int N = decltype(n_c)::value, NPC = decltype(npc_c)::value, ODD = decltype(odd_c)::value;
      constexpr bool OPEN = ((NPC - ODD) & 1) != 0, CLOSE = decltype(close_c)::value != 0;
      float acc[N / 2];
      auto taps = [&](auto ks_c) {
        uint32_t accumulate = 0;
        for (int g = ch.grp0; g < ch.grp0 + ch.ngrp; ++g) {
          if (blk_group_is_padding(p, g, tidx, oy_tile, ox0)) continue;
          ra.wait_full();
          const uint32_t a_hi0 = ptx::smem_u32(a_ring + (size_t)ra.slot * kBlkAStage) + (uint32_t)(wg * 64 * 128);
          for (int j = 0; j < p.gsize[g]; ++j) {
            rb.wait_full();
            const bool last = j + 1 == p.gsize[g];
            const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)rb.slot * kBlkBStage);
            // tap j of the group: shifted by j image rows
            issue(n_c, ks_c, acc, a_hi0 + (uint32_t)(j * 16 * 128), b_hi, ch.ks_first, accumulate,
                  last && !with_proj && !last_chain ? ra.slot : -1, rb.slot);
            accumulate = 1;
            rb.advance();
            if constexpr (decltype(first_c)::value != 0) {
              if (out_slot >= 0) {
                if (wtid == 0) { ptx::bulk_wait_read0(); ptx::mbar_arrive(&ra.empty[out_slot]); }
                out_slot = -1;
              }
            }
          }
          if (with_proj) {                       // the 1x1 projection of x reads the same stage (one group, centre tap)
            rb.wait_full();
            issue(BlkC<64>{}, ks_c, acc3, a_hi0, ptx::smem_u32(b_ring + (size_t)rb.slot * kBlkBStage), p.res.ks_first, 0u,
                  last_chain ? -1 : ra.slot, rb.slot);
            rb.advance();
          }
          if (last_chain) stage = ra.slot;
          ra.advance();
        }
      };
      switch (ch.ks_end - ch.ks_first) {
        case 1: taps(BlkC<1>{}); break;
        case 2: taps(BlkC<2>{}); break;
        case 3: taps(BlkC<3>{}); break;
        default: taps(BlkC<4>{}); break;
      }
      wg::wait<0>();                             // also: the previous chain's aggregation has read its P registers
      pend.release();
      // piece k of the chain = its 8-column group k = P piece pc0 + k: relu(acc + bias) split to bf16 hi / lo.
      // Accumulator entries (4 k + 2 h, +1) -- row row0 + 8 h, columns 8 k + cq, +1 -- are bf16x2 register h of the piece
      uint32_t f_hi[NPC][2], f_lo[NPC][2];
#pragma unroll
      for (int k = 0; k < NPC; ++k) {
        const float* bias = hb + (ch.pc0 + k) * 8 + cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float x0 = fmaxf(acc[4 * k + 2 * h] + bias[0], 0.f);
          const float x1 = fmaxf(acc[4 * k + 2 * h + 1] + bias[1], 0.f);
          ptx::split_hilo(x0, x1, f_hi[k][h], f_lo[k][h]);
        }
      }
      wg::fence();
      if constexpr (ODD) {                       // complete the step the previous chain began
        const uint32_t a_hi[4] = {carry_hi[0], carry_hi[1], f_hi[0][0], f_hi[0][1]};
        const uint32_t a_lo[4] = {carry_lo[0], carry_lo[1], f_lo[0][0], f_lo[0][1]};
        agg_step(agg_next++, a_hi, a_lo);
      }
#pragma unroll
      for (int k = ODD; k + 1 < NPC; k += 2) {
        const uint32_t a_hi[4] = {f_hi[k][0], f_hi[k][1], f_hi[k + 1][0], f_hi[k + 1][1]};
        const uint32_t a_lo[4] = {f_lo[k][0], f_lo[k][1], f_lo[k + 1][0], f_lo[k + 1][1]};
        agg_step(agg_next++, a_hi, a_lo);
      }
      if constexpr (OPEN && CLOSE) {             // the last piece of P: the other half of its step is zero
        const uint32_t a_hi[4] = {f_hi[NPC - 1][0], f_hi[NPC - 1][1], 0u, 0u};
        const uint32_t a_lo[4] = {f_lo[NPC - 1][0], f_lo[NPC - 1][1], 0u, 0u};
        agg_step(agg_next++, a_hi, a_lo);
      } else if constexpr (OPEN) {
        carry_hi[0] = f_hi[NPC - 1][0]; carry_hi[1] = f_hi[NPC - 1][1];
        carry_lo[0] = f_lo[NPC - 1][0]; carry_lo[1] = f_lo[NPC - 1][1];
      }
      wg::commit();
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
    ptx::mbar_wait(w_agg_full, 0);
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
      // ---------- the chains, each followed by the aggregation steps its pieces of P complete
      agg_next = 0;
      if constexpr (LAYOUT == kBlkThreePaths) {
        run_chain(BlkC<1>{}, BlkC<48>{}, BlkC<5>{}, BlkC<0>{}, BlkC<0>{}, p.chain[0], tidx, oy_tile, ox0, false, false);
        run_chain(BlkC<0>{}, BlkC<48>{}, BlkC<5>{}, BlkC<1>{}, BlkC<0>{}, p.chain[1], tidx, oy_tile, ox0, false, false);
        run_chain(BlkC<0>{}, BlkC<48>{}, BlkC<5>{}, BlkC<0>{}, BlkC<1>{}, p.chain[2], tidx, oy_tile, ox0, p.has_res_proj != 0, true);
      } else {
        run_chain(BlkC<1>{}, BlkC<64>{}, BlkC<8>{}, BlkC<0>{}, BlkC<0>{}, p.chain[0], tidx, oy_tile, ox0, false, false);
        run_chain(BlkC<0>{}, BlkC<32>{}, BlkC<4>{}, BlkC<0>{}, BlkC<0>{}, p.chain[1], tidx, oy_tile, ox0, p.has_res_proj != 0, true);
      }
      wg::wait<0>();
      pend.release();
      // ---------- output: relu(acc2 + bias) + residual, two channels per 8-column group and row, into the staging
      // stage: row r of this warpgroup's 64 at r * 128 bytes of each plane, 16-byte chunk g8 at chunk g8 ^ (r & 7).
      // For the identity residual those bytes hold x (path 2's 1x1 loaded channels 0..63 of these pixels), and each
      // thread reads exactly the words it then overwrites
      unsigned char* st_hi = a_ring + (size_t)stage * kBlkAStage;
      unsigned char* st_lo = st_hi + kBlkAStage / 2;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        const bool inside = oy_tile + (row >> 4) < p.H && ox0 + (row & 15) < p.W;
#pragma unroll
        for (int g8 = 0; g8 < 8; ++g8) {
          const int c = 8 * g8 + cq;
          const uint32_t off = (uint32_t)(row * 128 + ((g8 ^ (row & 7)) << 4) + 2 * cq);
          uint32_t* w_hi = reinterpret_cast<uint32_t*>(st_hi + off);
          uint32_t* w_lo = reinterpret_cast<uint32_t*>(st_lo + off);
          float v0 = fmaxf(acc2[4 * g8 + 2 * h] + wb[c], 0.f);
          float v1 = fmaxf(acc2[4 * g8 + 2 * h + 1] + wb[c + 1], 0.f);
          if (p.has_res_proj) {
            v0 += acc3[4 * g8 + 2 * h] + wb[64 + c];
            v1 += acc3[4 * g8 + 2 * h + 1] + wb[64 + c + 1];
          } else {                               // identity residual: the block's input planes
            const float2 r = ptx::join_hilo(*w_hi, *w_lo);
            v0 += r.x;
            v1 += r.y;
          }
          uint32_t hw, lw;
          ptx::split_hilo(v0, v1, hw, lw);
          *w_hi = hw;
          *w_lo = lw;
          if (p.sum_part && inside) { sacc[2 * g8] += v0; sacc[2 * g8 + 1] += v1; }
        }
      }
      ptx::fence_proxy_async();                  // the generic-proxy writes are visible to the TMA stores
      ptx::bar_sync(1 + wg, 128);                // every row of this warpgroup's half is written
      if (wtid == 0) {                           // image rows oy_tile + 4 wg .. + 3: the map clips the ragged edges
        const uint32_t src = ptx::smem_u32(st_hi) + (uint32_t)(wg * 64 * 128);
        ptx::tma_store_4d(&tm_o_hi, src, 0, ox0, oy_tile + kBlkStoreRows * wg, img);
        ptx::tma_store_4d(&tm_o_lo, src + kBlkAStage / 2, 0, ox0, oy_tile + kBlkStoreRows * wg, img);
        ptx::bulk_commit();
      }
      out_slot = stage;
    }
    if (p.sum_part && sum_img >= 0) flush_sums(sum_img);
    if (wtid == 0) ptx::bulk_wait0();            // the last tile's outputs are written before the CTA exits
  }
}
}  // namespace stp3

using namespace stp3;

extern "C" size_t stp3_block_fused_scratch_bytes(int n_img) {
  return (size_t)num_sms() * 8 * (size_t)(n_img > 0 ? n_img : 0) * 64 * sizeof(float);
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
  {
    const stp3_block_chain& last = d->chain[d->n_chain - 1];
    STP3_CHECK_ARG(last.src == 1 && last.n_taps == 1 && (d->has_res_proj || last.cin_off == 0),
                   "the last chain is the 1x1 of x (its activation stage stages the output tile and, without a projection, "
                   "holds the identity residual: x's channels 0..63)");
  }
  auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
  STP3_CHECK_ARG(al32(y_hi) && al32(y_lo) && al32(x_hi) && al32(x_lo), "planes must be 32-byte aligned");

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
    const BlkChain& last = p.chain[p.n_chain - 1];
    STP3_CHECK_ARG(last.src == 1 && last.ntaps == 1 && last.cin_off == p.res.cin_off &&
                   last.ks_first == p.res.ks_first && last.ks_end == p.res.ks_end,
                   "the projection shares the last chain's activations: that chain is the 1x1 of x over the same channels");
  } else {
    p.res = p.chain[0];
  }
  // P: chain c produces pieces pc0 .. pc0 + npc - 1 (its 8-column groups 0 .. npc - 1), in chain order; zeros after
  static const int kShapes[2][kBlkMaxChains][2] = {{{48, 5}, {48, 5}, {48, 5}}, {{64, 8}, {32, 4}, {0, 0}}};
  const int layout = p.n_chain == 3 ? kBlkThreePaths : kBlkDiagPair;
  int pp = 0;
  for (int c = 0; c < p.n_chain; ++c) {
    BlkChain& ch = p.chain[c];
    ch.pc0 = pp;
    int npc = 0;
    while (pp < 16 && d->piece_col[pp] >= 0 && d->piece_col[pp] == ch.tmem_col + 8 * npc && 8 * npc < ch.n_mma) { ++pp; ++npc; }
    STP3_CHECK_ARG(p.n_chain >= 2 && ch.n_mma == kShapes[layout][c][0] && npc == kShapes[layout][c][1],
                   "chain %d of %d: (N, pieces of P) = (%d, %d) is not a compiled chain layout", c, p.n_chain, ch.n_mma, npc);
  }
  for (; pp < 16; ++pp) STP3_CHECK_ARG(d->piece_col[pp] < 0, "piece %d of P: the chains' pieces are consecutive, zeros follow", pp);
  // every descriptor check comes before the driver lookup: a bad descriptor is reported as such without a GPU
  if (!tmap_encode_fn()) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
  p.hid_bias = hid_bias; p.img_bias = img_bias; p.res_bias = res_bias;

  CUtensorMap tm[4], tm_w, tm_o[2];
  const void* planes[4] = {mid_hi, mid_lo, x_hi, x_lo};
  for (int i = 0; i < 4; ++i) {
    const CUresult r = encode_act_5d(&tm[i], planes[i], i < 2 ? d->mid_cstride : d->x_cstride, d->W, d->H, d->T, d->B,
                                     16, kBlkBoxRows, 1);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation %d) failed: %d", i, (int)r);
  }
  {
    const CUresult r = encode_rows_2d(&tm_w, w, (long long)blk * 256, 8);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  }
  void* outs[2] = {y_hi, y_lo};
  for (int i = 0; i < 2; ++i) {       // channels [0, 64) of the output window; one box = one warpgroup's 4 x 16 pixels
    const CUresult r = encode_out_4d(&tm_o[i], outs[i], d->out_cstride, 64, d->W, d->H, p.n_img, 16, kBlkStoreRows);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(output %d) failed: %d", i, (int)r);
  }
  auto kern = layout == kBlkThreePaths ? block_fused_kernel<kBlkThreePaths> : block_fused_kernel<kBlkDiagPair>;
  STP3_CUDA_OK(layout == kBlkThreePaths ? set_max_dynamic_smem<block_fused_kernel<kBlkThreePaths>>((int)BlkSmem::bytes)
                                        : set_max_dynamic_smem<block_fused_kernel<kBlkDiagPair>>((int)BlkSmem::bytes));
  const int n_sm = num_sms();
  const unsigned grid = (unsigned)(nt < n_sm ? nt : n_sm);
  p.sum_part = nullptr;
  if (col_sums) {
    const size_t need = (size_t)grid * 8 * p.n_img * 64 * sizeof(float);
    STP3_CHECK_ARG(scratch && scratch_bytes >= need, "col_sums: scratch missing or smaller than stp3_block_fused_scratch_bytes()");
    p.sum_part = static_cast<float*>(scratch);
    STP3_CUDA_OK(cudaMemsetAsync(p.sum_part, 0, need, stream));
  }
  // The back-to-back kernels never execute griddepcontrol.launch_dependents, so their dependents start only when the
  // grid has completed.  Each of them needs a whole SM; an early trigger would let a chain block_fused -> col_sum_reduce
  // -> pool_bias -> aspp_fused be resident at once, and such a chain was seen to stop making progress.  The kernel itself
  // still starts early behind its predecessor (griddepcontrol.wait before it reads what that predecessor wrote).
  STP3_CUDA_OK(launch_pdl(kPdlFused, kern, dim3(grid), dim3(kBlkThreads), BlkSmem::bytes, stream, tm[0], tm[1], tm[2],
                          tm[3], tm_w, tm_o[0], tm_o[1], p));
  STP3_CUDA_OK(cudaGetLastError());
  if (col_sums) return launch_col_sum_reduce(p.sum_part, (int)grid * 8, p.n_img, col_sums, stream);
  return STP3_OK;
}
