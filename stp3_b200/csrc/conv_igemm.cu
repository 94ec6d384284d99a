// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, register accumulators), operands staged by TMA.
//
// One kernel family covers every dense layer of the hot path (1x1x1, causal (2,3,3) / (1,3,3) 3-D, dilated 3x3,
// 7x7 stride 2, 3x3 / 1x1 stride 2): a convolution is a sum over taps of [pixels x Cin] . [Cin x Cout] GEMMs whose
// A operand is a shifted (strided, zero-padded) window of the channels-last activation tensor -- exactly what a
// 5-D TMA box with out-of-bounds zero fill delivers.
//
// Precision: fp32 tensors are carried as two bf16 planes (hi = bf16(x), lo = bf16(x - hi)); every product is
// evaluated as hi*hi + hi*lo + lo*hi on the bf16 tensor pipe with fp32 accumulation (error ~2^-16 per product
// instead of 2^-8), which keeps 25 stacked layers inside the 1e-3 parity bar.  Eval-mode BatchNorm is folded into
// the weights/bias on the host; bias, per-image bias (pyramid-pool / ASPP-pool / ego-motion branches), ReLU,
// residual add and the concat offset are fused in the epilogue.
//
//   tile     : 128 output pixels (8 x 16 of one image) x BN output channels (64 / 128; 256 runs as two launches)
//   K loop   : taps x (Cin / 64); TMA brings A_hi, A_lo (128 or 160 pixel rows x 64 bf16, 128B-swizzled; one load
//              serves the three dy taps of a 3x3) and B_hi, B_lo (BN x 64; small weight tensors stay resident in
//              smem) through separate rings; each warpgroup issues 4 (K = 16) x 3 wgmma per tap for its 64 rows
//   CTA      : persistent, one per SM, walks tiles blockIdx.x + i*gridDim.x
//   warps    : 0..7 = two MMA warpgroups (rows 0..63 / 64..127 of the tile) that also run the epilogue (registers ->
//              shared accumulator tile -> global), 8 = TMA producer, which keeps loading the next tile's operands
//              while the epilogue drains
//
// Reference layers: stp3/layers/temporal.py:252-489, stp3/layers/convolutions.py:183-280, stp3/models/decoder.py.
#include <cuda_bf16.h>

#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kEpiWarps = 8;                     // two warps per 32-row quarter of the tile, each owning half of the columns
constexpr int kConvThreads = kEpiWarps * 32 + 32;
constexpr int kSubH = 8, kTileW = 16;           // one tile = 8 x 16 pixels = 128 accumulator rows
constexpr int kBK = 64;                         // channels per K step (one 128-byte swizzle row of bf16)
constexpr int kMaxTaps = 49;
constexpr int kMaxAStages = 4, kMaxBStages = 8;
constexpr int kMaxHeadOut = 8;

struct ConvParams {
  int n_img, T, t0, Ho, Wo;
  int T_total;              // frames of the input tensor
  int H, W;                 // input image size
  int skip_t;               // skip tap groups whose window lies entirely in the zero padding for the whole tile (frame
                            // outside [0, T_total): causal convs at t = 0; rows / columns outside the image: dilated convs)
  int tiles_x, tiles_y, n_tiles;
  int stride;
  int kblocks;              // Cin / 64 of this convolution
  int cin_off;              // first input channel inside the (wider) input tensor, multiple of 64
  int ntaps;
  int ks_first, ks_end;     // K = 16 steps that carry data: [ks_first, 4) of the first K block, [0, ks_end) of the last
                            // (channels outside are zero padding of a narrow convolution: neither multiplied nor needed)
  // taps that share one activation load: consecutive taps with the same (dt, dx) whose dy advance by the stride read
  // the same strided rows shifted by one OUTPUT row each (the three dy taps of a 3x3; dy = -3,-1,1,3 / -2,0,2 of the
  // stride-2 7x7), so one box of tile_rows + gmax - 1 rows serves the whole group
  int n_groups, gmax;
  unsigned char gstart[kMaxTaps], gsize[kMaxTaps];
  int a_plane_bytes;        // bytes of one activation plane of a stage = box_h * 16 px * 128 B
  int n_mma;                // output columns the MMAs compute (multiple of 16, <= BN): columns beyond the convolution's
                            // real Cout have zero weights and bias, so they are neither loaded nor multiplied
  int b_rows;               // weight rows per plane part in shared memory: n_mma, or BN for full-K launches (the
                            // wgmma N is then BN; rows beyond n_mma are never loaded and their columns never read)
  int b_tile_bytes;         // shared-memory bytes of one K step's weights (hi and lo parts)
  int b_load_bytes;         // bytes TMA brings per K step: 2 * n_mma rows
  int w_rows;               // rows per (tap, kb, plane) block of the packed weight tensor (the convolution's padded Cout)
  int w_row_off;            // first row of this launch inside that block (a 256-channel conv runs as two launches)
  signed char tap[kMaxTaps][4];   // (dt, dy, dx): input coordinate = output coordinate * stride + d
  const float* bias;        // [BN]
  const float* img_bias;    // [n_img][img_bias_stride] or null (replaces bias)
  int img_bias_stride;
  int relu;
  int res_mode;             // 0 none, 1 residual added before the activation, 2 after
  const __nv_bfloat16* res_hi;
  const __nv_bfloat16* res_lo;
  int res_cstride, res_coff;
  __nv_bfloat16* out_hi;    // channels-last (n_img, Ho, Wo, out_cstride), may be null when out_f32 is used
  __nv_bfloat16* out_lo;
  int out_cstride, out_coff, n_store;
  int vec256;               // bit 0: output rows / windows are 32-byte aligned (256-bit stores), bit 1: residual likewise
  float* out_f32;           // optional (n_img, n_valid, Ho, Wo) fp32, the reference's NCHW layout
  int n_valid, f32_coff;    // channel offset of this launch inside out_f32
  int f32_nhwc;             // out_f32 is channels-last (n_img, Ho, Wo, n_valid): 16 channels of a pixel = two 32-byte stores
  int sigmoid;              // apply to out_f32 (instance_center head)
  int na_stages, nb_stages; // smem ring depths chosen by the host
  int b_resident;           // all weight tiles of the convolution stay in shared memory for the CTA's lifetime
  // fused 1x1 "head" on the activated tile: out_k = head_b[k] + sum_c head_w[k][c] * y[c]  (decoder heads 3x3 -> 1x1)
  int head_ko;              // 0 = off, else 1..8 outputs
  const float* head_w;      // [head_ko][BN]
  const float* head_b;      // [head_ko]
  float* head_out[8];       // plane of output k for image 0 (fp32, (Ho, Wo))
  long long head_img_stride[8];   // elements between consecutive images for output k
  int head_sigmoid_mask;    // bit k: sigmoid on output k
  // second destination (BN = 128): output columns [64, 128) go to another tensor with their own activation flag -- two
  // 64-column convolutions that read the same input run as one launch and read it once
  __nv_bfloat16* out2_hi;
  __nv_bfloat16* out2_lo;
  int out2_cstride, out2_coff, n_store2, relu2;
  // per-image column sums of the activated output (the consumer's pooling branches need sum over H*W): every epilogue
  // warp keeps running sums of its pixels in registers and writes one partial row per (CTA, row quarter, image) --
  // plain stores, fixed order: deterministic.  BN = 64 only.  sum_part: [gridDim.x][4][n_img][BN], zeroed by the host.
  float* sum_part;
};

// STACK (BN = 64 only): the hi and lo weight planes of a K step form ONE B operand of 2*BN rows, so a product is two
// MMAs instead of three -- A_hi x [W_hi; W_lo] (N = 2*BN) and A_lo x W_hi (N = BN) -- and the activation tile is read
// from shared memory twice instead of three times.  The accumulator has 2*BN columns; the epilogue adds columns c and
// n_mma + c.
template <int BN, bool STACK = false>
struct ConvSmem {
  static constexpr int kAccCols = STACK ? 2 * BN : BN;                 // accumulator columns
  static constexpr int kAccStride = kAccCols + 4;                      // floats per row of the shared accumulator tile
  static constexpr size_t tail_bytes() {
    return (1 + kMaxHeadOut) * BN * sizeof(float) + kMaxHeadOut * 128 * sizeof(float) + kEpiWarps * 64 * sizeof(float) +
           (size_t)128 * kAccStride * sizeof(float) + (2 * kMaxAStages + 2 * kMaxBStages + 8) * 8;
  }
};

// true if every input element the tap group touches for this tile is zero padding (same answer in the producer and
// the MMA warpgroups: it looks at the whole tile)
__device__ __forceinline__ bool group_is_padding(const ConvParams& p, int grp, int tidx, int oy_tile, int ox0, int tile_h) {
  const int tap0 = p.gstart[grp];
  const int t = tidx + p.tap[tap0][0];
  const int ylo = oy_tile * p.stride + p.tap[tap0][1];
  const int yhi = (oy_tile + tile_h - 1 + p.gsize[grp] - 1) * p.stride + p.tap[tap0][1];
  const int xlo = ox0 * p.stride + p.tap[tap0][2];
  const int xhi = (ox0 + kTileW - 1) * p.stride + p.tap[tap0][2];
  return t < 0 || t >= p.T_total || yhi < 0 || ylo >= p.H || xhi < 0 || xlo >= p.W;
}

__device__ __forceinline__ void ld_acc16(const float* src, uint32_t (&r)[16]) {   // 16 consecutive fp32, 16-byte aligned
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + 4 * g);
    r[4 * g] = v.x; r[4 * g + 1] = v.y; r[4 * g + 2] = v.z; r[4 * g + 3] = v.w;
  }
}

// Persistent, warp-specialised implicit-GEMM convolution.
//   * A CTA walks output tiles blockIdx.x + i*gridDim.x; a tile is 8x16 pixels = 128 accumulator rows, 64 per warpgroup.
//   * Activations and weights travel through separate shared-memory rings filled by one producer warp.  For 3x3 /
//     stride 1 / dilation 1 kernels one activation load of 10 image rows serves the three dy taps: their A operands are
//     the same smem tile at row offsets 0, 16, 32 (2 KB steps keep the 1024-byte swizzle alignment).
//   * wgmma groups are committed per tap; a ring slot is released once the group after the one that read it has been
//     issued and the reading group has retired (wgmma.wait_group 1), so the tensor pipe always has the next tap queued.
//   * At the end of a tile the accumulators go to a shared [128 rows][columns] fp32 tile; the epilogue gives every
//     thread one pixel (row) and half of the columns.
// FULLK: every K = 16 step of every K block carries data (ks_first == 0, ks_end == 4).  Then a tap is a branch-free run
// of wgmma with N fixed at compile time (BN, 2 * BN for the stacked operand), which ptxas pipelines; any branch around
// the MMAs (skipped K steps, an N chosen at run time) makes it serialise them.
template <int BN, bool STACK, bool FULLK>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_w, const ConvParams p) {
  using S = ConvSmem<BN, STACK>;
  static_assert(!STACK || BN == 64, "stacked weight operand: BN = 64 only");
  constexpr int kAccRegs = S::kAccCols / 2;        // accumulator registers per thread (64 rows x kAccCols per warpgroup)
  const int kBRows = p.b_rows;
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte alignment for the 128-byte swizzle; plain offset arithmetic keeps the pointer in the shared state space
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int k_iters = p.ntaps * p.kblocks;
  const bool resident = p.b_resident != 0;
  const int a_stage_bytes = 2 * p.a_plane_bytes;
  unsigned char* a_ring = smem;
  unsigned char* b_ring = a_ring + (size_t)p.na_stages * a_stage_bytes;            // ring, or the resident weights
  float* s_bias = reinterpret_cast<float*>(b_ring + (size_t)(resident ? k_iters : p.nb_stages) * p.b_tile_bytes);
  float* s_head = s_bias + BN;                    // [kMaxHeadOut][BN]
  float* s_hx = s_head + kMaxHeadOut * BN;        // [kMaxHeadOut][128] head partials handed between column halves
  float* s_wb = s_hx + kMaxHeadOut * 128;         // [kEpiWarps][64] per-image bias slice of each epilogue warp
  float* s_acc = s_wb + kEpiWarps * 64;           // [128][kAccStride] accumulator tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_acc + 128 * S::kAccStride);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kMaxAStages;
  uint64_t* b_full = a_empty + kMaxAStages;
  uint64_t* b_empty = b_full + kMaxBStages;
  uint64_t* bres_bar = b_empty + kMaxBStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // Programmatic dependent launch: the next conv of the stream may set up (barriers, resident weights) on SMs this grid
  // has left; this grid's own set-up ran while its predecessor drained.  Only module constants (bias, weights, head
  // weights) are read before griddep_wait().
  ptx::griddep_launch_dependents();
  if (warp == kEpiWarps && lane == 0) {
    ptx::prefetch_tmap(&tm_a_hi); ptx::prefetch_tmap(&tm_a_lo); ptx::prefetch_tmap(&tm_w);
    for (int i = 0; i < p.na_stages; ++i) { ptx::mbar_init(&a_full[i], 1); ptx::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < p.nb_stages; ++i) { ptx::mbar_init(&b_full[i], 1); ptx::mbar_init(&b_empty[i], 2); }
    ptx::mbar_init(bres_bar, 1);
    ptx::fence_mbar_init();
  }
  for (int i = threadIdx.x; i < BN; i += blockDim.x) s_bias[i] = p.bias[i];
  for (int i = threadIdx.x; i < p.head_ko * BN; i += blockDim.x) s_head[i] = p.head_w[i];
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int n_groups = p.n_groups;
  const int tile_h = kSubH;

  if (warp == kEpiWarps) {
    // ===================== TMA producer (whole warp walks the loops; one elected lane issues) =====================
    // load_b: the weight tile of K step `it` into `dst` (called by the elected lane; transaction bytes on `bar`)
    auto load_b = [&](unsigned char* dst, int it, uint64_t* bar) {
      const int row_hi = (it * 2) * p.w_rows + p.w_row_off, row_lo = row_hi + p.w_rows;
      ptx::tma_load_2d(dst, &tm_w, bar, 0, row_hi);                       // [W_hi; W_lo], also the stacked operand
      ptx::tma_load_2d(dst + kBRows * kBK * 2, &tm_w, bar, 0, row_lo);
    };
    if (resident && ptx::elect_one_sync()) {
      ptx::mbar_arrive_expect_tx(bres_bar, (uint32_t)(k_iters * p.b_load_bytes));
      for (int it = 0; it < k_iters; ++it) load_b(b_ring + (size_t)it * p.b_tile_bytes, it, bres_bar);
    }
    __syncwarp();
    ptx::griddep_wait();                        // activations come from the preceding kernel
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy0 = (rem / p.tiles_x) * tile_h, ox0 = (rem % p.tiles_x) * kTileW;
      const int bidx = img / p.T, tidx = p.t0 + img % p.T;
      for (int grp = 0; grp < n_groups; ++grp) {
        const int tap0 = p.gstart[grp], gsz = p.gsize[grp];
        const int x = ox0 * p.stride + p.tap[tap0][2];
        const int y = oy0 * p.stride + p.tap[tap0][1];
        const int t = tidx + p.tap[tap0][0];
        if (p.skip_t && group_is_padding(p, grp, tidx, oy0, ox0, tile_h)) continue;
        for (int kb = 0; kb < p.kblocks; ++kb) {
          ptx::mbar_wait(&a_empty[as], aph ^ 1);
          if (ptx::elect_one_sync()) {
            unsigned char* sa = a_ring + (size_t)as * a_stage_bytes;
            const int c = p.cin_off + kb * kBK;
            ptx::mbar_arrive_expect_tx(&a_full[as], (uint32_t)a_stage_bytes);
            ptx::tma_load_5d(sa, &tm_a_hi, &a_full[as], c, x, y, t, bidx);
            ptx::tma_load_5d(sa + p.a_plane_bytes, &tm_a_lo, &a_full[as], c, x, y, t, bidx);
          }
          __syncwarp();
          if (++as == p.na_stages) { as = 0; aph ^= 1; }
          if (!resident) {
            for (int j = 0; j < gsz; ++j) {
              const int it = (tap0 + j) * p.kblocks + kb;          // [tap][kb][plane][rows] blocks of 64-wide rows
              ptx::mbar_wait(&b_empty[bs], bph ^ 1);
              if (ptx::elect_one_sync()) {
                ptx::mbar_arrive_expect_tx(&b_full[bs], (uint32_t)p.b_load_bytes);
                load_b(b_ring + (size_t)bs * p.b_tile_bytes, it, &b_full[bs]);
              }
              __syncwarp();
              if (++bs == p.nb_stages) { bs = 0; bph ^= 1; }
            }
          }
        }
      }
    }
  } else {
    // ===================== two MMA warpgroups, then the epilogue =====================
    const int wg = warp >> 2;                    // warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float accr[kAccRegs];
    int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
    if (resident) ptx::mbar_wait(bres_bar, 0);
    // the accumulator of `tile` over every tap and K block -> s_acc
    auto mma_tile = [&](int tile) {
      const int tidx = p.t0 + (tile / tiles_per_img) % p.T;
      const int rem_m = tile % tiles_per_img;
      const int oy_m = (rem_m / p.tiles_x) * tile_h, ox_m = (rem_m % p.tiles_x) * kTileW;
      uint32_t accumulate = 0;
      int pend_a = -1, pend_b = -1;              // ring slots read by the last committed wgmma group
      auto release = [&]() {
        if (wg_leader) {
          if (pend_a >= 0) ptx::mbar_arrive(&a_empty[pend_a]);
          if (pend_b >= 0) ptx::mbar_arrive(&b_empty[pend_b]);
        }
        pend_a = pend_b = -1;
      };
      for (int grp = 0; grp < n_groups; ++grp) {
        if (p.skip_t && group_is_padding(p, grp, tidx, oy_m, ox_m, tile_h)) continue;
        const int tap0 = p.gstart[grp], gsz = p.gsize[grp];
        for (int kb = 0; kb < p.kblocks; ++kb) {
          ptx::mbar_wait(&a_full[as], aph);
          const int k_begin = kb == 0 ? p.ks_first : 0, k_end = kb == p.kblocks - 1 ? p.ks_end : kBK / 16;
          const uint32_t a_hi0 = ptx::smem_u32(a_ring + (size_t)as * a_stage_bytes) + (uint32_t)(wg * 64 * 128);
          for (int j = 0; j < gsz; ++j) {
            const int it = (tap0 + j) * p.kblocks + kb;
            uint32_t b_hi;
            if (resident) {
              b_hi = ptx::smem_u32(b_ring + (size_t)it * p.b_tile_bytes);
            } else {
              ptx::mbar_wait(&b_full[bs], bph);
              b_hi = ptx::smem_u32(b_ring + (size_t)bs * p.b_tile_bytes);
            }
            // stacked: db_hi = [W_hi; W_lo] (2 * b_rows rows), db_lo = W_hi alone
            const uint64_t db_hi = wg::desc_k_sw128(b_hi);
            const uint64_t db_lo = wg::desc_k_sw128(b_hi + (STACK ? 0 : kBRows * kBK * 2));
            // this warpgroup's 64 rows of the tile, shifted by j image rows inside the loaded box
            const uint32_t a_hi = a_hi0 + (uint32_t)(j * kTileW * 128);
            const uint64_t da_hi = wg::desc_k_sw128(a_hi), da_lo = wg::desc_k_sw128(a_hi + p.a_plane_bytes);
            wg::fence();
            if constexpr (FULLK) {
#pragma unroll
              for (int k = 0; k < kBK / 16; ++k) {
                const uint64_t koff = (uint64_t)((k * 16 * 2) >> 4);   // advance 16 bf16 = 32 bytes along K
                const uint32_t acc0 = accumulate | (uint32_t)(k > 0);
                if constexpr (STACK) {
                  wg::mma_bf16<2 * BN>(accr, da_hi + koff, db_hi + koff, acc0);                // A_hi x [W_hi; W_lo]
                  wg::mma_bf16<BN>(accr, da_lo + koff, db_lo + koff, 1);                       // A_lo x W_hi
                } else {
                  wg::mma_bf16<BN>(accr, da_hi + koff, db_hi + koff, acc0);
                  wg::mma_bf16<BN>(accr, da_hi + koff, db_lo + koff, 1);
                  wg::mma_bf16<BN>(accr, da_lo + koff, db_hi + koff, 1);
                }
              }
            } else {
#pragma unroll
              for (int k = 0; k < kBK / 16; ++k) {
                if (k < k_begin || k >= k_end) continue;               // K steps of pure channel padding
                const uint64_t koff = (uint64_t)((k * 16 * 2) >> 4);
                const uint32_t acc0 = accumulate | (uint32_t)(k > k_begin);
                if constexpr (STACK) {
                  wg::mma_bf16_n<2 * BN>(2 * p.n_mma, accr, da_hi + koff, db_hi + koff, acc0);
                  wg::mma_bf16_n<2 * BN>(p.n_mma, accr, da_lo + koff, db_lo + koff, 1);
                } else {
                  wg::mma_bf16_n<BN>(p.n_mma, accr, da_hi + koff, db_hi + koff, acc0);
                  wg::mma_bf16_n<BN>(p.n_mma, accr, da_hi + koff, db_lo + koff, 1);
                  wg::mma_bf16_n<BN>(p.n_mma, accr, da_lo + koff, db_hi + koff, 1);
                }
              }
            }
            wg::commit();
            wg::wait<1>();                         // the previous group has read its operands
            release();
            pend_b = resident ? -1 : bs;
            if (j + 1 == gsz) pend_a = as;
            accumulate = 1;
            if (!resident) { if (++bs == p.nb_stages) { bs = 0; bph ^= 1; } }
          }
          if (++as == p.na_stages) { as = 0; aph ^= 1; }
        }
      }
      wg::wait<0>();
      release();
      // registers -> s_acc (columns the MMAs computed)
      const int ncols = STACK ? 2 * kBRows : kBRows;
      const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < kAccRegs; i += 2) {
        const int col = 8 * (i >> 2) + 2 * (lane & 3);
        if (col < ncols) {
          const int row = row0 + 8 * ((i >> 1) & 1);
          *reinterpret_cast<float2*>(s_acc + (size_t)row * S::kAccStride + col) = make_float2(accr[i], accr[i + 1]);
        }
      }
      ptx::bar_sync(5, kEpiWarps * 32);
    };
    // ----- epilogue: shared accumulator tile -> registers -> global
    const int e = warp;
    const int q = warp & 3;                      // 32-row quarter of the tile this warp drains
    const int half = e >> 2;                     // which half of the BN columns this warp handles
    constexpr int kColsPerWarp = BN / 2;
    const int col0 = half * kColsPerWarp;
    const int r = q * 32 + lane;                 // row of the tile = output pixel
    // destination of this warp's columns (the upper column half may belong to a second tensor)
    const bool second = BN == 128 && half == 1 && p.out2_hi != nullptr;
    __nv_bfloat16* const d_hi = second ? p.out2_hi : p.out_hi;
    __nv_bfloat16* const d_lo = second ? p.out2_lo : p.out_lo;
    const int d_cstride = second ? p.out2_cstride : p.out_cstride;
    const int d_coff = second ? p.out2_coff - 64 : p.out_coff;          // d_coff + column = channel in the destination
    const int d_nstore = second ? 64 + p.n_store2 : p.n_store;
    const bool d_relu = (second ? p.relu2 : p.relu) != 0;
    const bool d_vec = ((p.vec256 >> (second ? 2 : 0)) & 1) != 0;
    constexpr bool kSums = BN == 64;              // column sums need kColsPerWarp (= 32) accumulators per thread
    float sacc[kSums ? 32 : 1];
#pragma unroll
    for (int i = 0; i < (kSums ? 32 : 1); ++i) sacc[i] = 0.f;
    int sum_img = -1;
    auto flush_sums = [&](int img_) {             // 32 lanes x 32 columns -> lane l holds column col0 + l (halving butterfly)
      if constexpr (kSums) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          const bool upper = (lane & off) != 0;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            if (i < off) {
              const float send = upper ? sacc[i] : sacc[i + off];
              const float keep = upper ? sacc[i + off] : sacc[i];
              sacc[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
          }
        }
        p.sum_part[(((size_t)blockIdx.x * 4 + q) * p.n_img + img_) * BN + col0 + lane] = sacc[0];
#pragma unroll
        for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
      }
    };
    ptx::griddep_wait();                          // residual / per-image bias reads and every global write come after
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_t = (rem / p.tiles_x) * kSubH, ox = (rem % p.tiles_x) * kTileW + (r & 15);
      if (kSums && p.sum_part && img != sum_img) {      // tiles come in image order: hand the finished image over
        if (sum_img >= 0) flush_sums(sum_img);
        sum_img = img;
      }
      // latency hiding: the residual of the first chunk and this warp's slice of the per-image bias are requested
      // before waiting for the accumulator; every later residual chunk is requested one chunk ahead
      uint32_t nh[8], nl[8];
      auto request_residual = [&](int j) {
        const int oy = oy_t + (r >> 4);
        if (oy < p.Ho && ox < p.Wo) {
          const size_t off = (((size_t)img * p.Ho + oy) * p.Wo + ox) * p.res_cstride + p.res_coff + col0 + j * 16;
          // coherent loads: the residual (like the per-image bias below) is written by a PRECEDING kernel that this grid
          // may overlap under programmatic dependent launch, so the read-only (.nc) path is not allowed for it
          if (p.vec256 & 2) {
            ptx::ld_global_v8(p.res_hi + off, nh);
            ptx::ld_global_v8(p.res_lo + off, nl);
          } else {
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              const uint4 h4 = ptx::ld_global_v4(reinterpret_cast<const uint4*>(p.res_hi + off) + g);
              const uint4 l4 = ptx::ld_global_v4(reinterpret_cast<const uint4*>(p.res_lo + off) + g);
              nh[4 * g] = h4.x; nh[4 * g + 1] = h4.y; nh[4 * g + 2] = h4.z; nh[4 * g + 3] = h4.w;
              nl[4 * g] = l4.x; nl[4 * g + 1] = l4.y; nl[4 * g + 2] = l4.z; nl[4 * g + 3] = l4.w;
            }
          }
        }
      };
      if (p.res_mode) request_residual(0);
      const float* bsrc = s_bias;                 // bias of column c at bsrc[c]
      if (p.img_bias) {
        const float* ib = p.img_bias + (size_t)img * p.img_bias_stride + col0;
        float* wb = s_wb + e * 64;
        __syncwarp();                             // every lane is done with the previous tile's slice
#pragma unroll
        for (int i = lane; i < kColsPerWarp; i += 32) wb[i] = *(reinterpret_cast<const volatile float*>(ib) + i);
        __syncwarp();
        bsrc = wb - col0;
      }
      mma_tile(tile);
      {
        const int oy = oy_t + (r >> 4);
        const bool valid = oy < p.Ho && ox < p.Wo;
        const size_t pix = ((size_t)img * p.Ho + oy) * p.Wo + ox;
        float hacc[kMaxHeadOut];
#pragma unroll
        for (int k = 0; k < kMaxHeadOut; ++k) hacc[k] = 0.f;
        const float* acc_row = s_acc + (size_t)r * S::kAccStride + col0;
#pragma unroll 1
        for (int j = 0; j < kColsPerWarp / 16; ++j) {
          const int cb = col0 + j * 16;              // first output channel of this chunk
          uint32_t acc[16];
          uint32_t acc2[16];                         // stacked operand: the hi x lo products live b_rows columns further
          const bool computed = cb < p.n_mma;        // columns beyond n_mma: zero weights, never multiplied
          if (computed) {
            ld_acc16(acc_row + j * 16, acc);
            if constexpr (STACK) ld_acc16(acc_row + kBRows + j * 16, acc2);
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) { acc[i] = 0u; acc2[i] = 0u; }
          }
          uint32_t rhw[8], rlw[8];                   // residual of this chunk (requested one chunk ago)
          if (p.res_mode) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { rhw[i] = nh[i]; rlw[i] = nl[i]; }
            const bool last_j = j + 1 == kColsPerWarp / 16;
            if (!last_j) request_residual(j + 1);
          }
          if (valid) {
            float v[16];
#pragma unroll
            for (int g = 0; g < 4; ++g) {          // bias: per-image slice (conv bias already folded in) or the conv's own
              const float4 b4 = *reinterpret_cast<const float4*>(bsrc + cb + 4 * g);
              if constexpr (STACK) {
                v[4 * g + 0] = (__uint_as_float(acc[4 * g + 0]) + __uint_as_float(acc2[4 * g + 0])) + b4.x;
                v[4 * g + 1] = (__uint_as_float(acc[4 * g + 1]) + __uint_as_float(acc2[4 * g + 1])) + b4.y;
                v[4 * g + 2] = (__uint_as_float(acc[4 * g + 2]) + __uint_as_float(acc2[4 * g + 2])) + b4.z;
                v[4 * g + 3] = (__uint_as_float(acc[4 * g + 3]) + __uint_as_float(acc2[4 * g + 3])) + b4.w;
              } else {
                v[4 * g + 0] = __uint_as_float(acc[4 * g + 0]) + b4.x;
                v[4 * g + 1] = __uint_as_float(acc[4 * g + 1]) + b4.y;
                v[4 * g + 2] = __uint_as_float(acc[4 * g + 2]) + b4.z;
                v[4 * g + 3] = __uint_as_float(acc[4 * g + 3]) + b4.w;
              }
            }
            if (p.res_mode) {
#pragma unroll
              for (int e2 = 0; e2 < 8; ++e2) {
                const float r0 = __uint_as_float(rhw[e2] << 16) + __uint_as_float(rlw[e2] << 16);
                const float r1 = __uint_as_float(rhw[e2] & 0xFFFF0000u) + __uint_as_float(rlw[e2] & 0xFFFF0000u);
                float& a0 = v[e2 * 2], &a1 = v[e2 * 2 + 1];
                if (p.res_mode == 1) { a0 += r0; a1 += r1; if (d_relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); } }
                else { if (d_relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); } a0 += r0; a1 += r1; }
              }
            } else if (d_relu) {
#pragma unroll
              for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
            }
            if (d_hi && cb < d_nstore) {
              __nv_bfloat16* ohp = d_hi + pix * d_cstride + d_coff + cb;
              __nv_bfloat16* olp = d_lo + pix * d_cstride + d_coff + cb;
              uint32_t hw[8], lw[8];
#pragma unroll
              for (int e2 = 0; e2 < 8; ++e2) {
                const float x0 = v[e2 * 2], x1 = v[e2 * 2 + 1];
                const uint32_t h = ptx::pack_bf16x2(x0, x1);                   // one cvt.rn.bf16x2.f32
                const float r0 = x0 - __uint_as_float(h << 16), r1 = x1 - __uint_as_float(h & 0xFFFF0000u);
                hw[e2] = h;
                lw[e2] = ptx::pack_bf16x2(r0, r1);
              }
              if (d_vec && cb + 16 <= d_nstore) {               // one full 32-byte sector per plane and lane
                ptx::st_global_v8(ohp, hw);
                ptx::st_global_v8(olp, lw);
              } else {
                reinterpret_cast<uint4*>(ohp)[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                reinterpret_cast<uint4*>(olp)[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                if (cb + 8 < d_nstore) {
                  reinterpret_cast<uint4*>(ohp)[1] = make_uint4(hw[4], hw[5], hw[6], hw[7]);
                  reinterpret_cast<uint4*>(olp)[1] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
                }
              }
            }
            if (p.out_f32 && p.f32_nhwc) {
              const int c0 = p.f32_coff + cb;
              float* dst = p.out_f32 + pix * p.n_valid + c0;
              if (c0 + 16 <= p.n_valid && (p.n_valid & 7) == 0) {          // rows are 32-byte aligned (host checks the base)
                ptx::st_global_v8f(dst, v);
                ptx::st_global_v8f(dst + 8, v + 8);
              } else {
#pragma unroll
                for (int i = 0; i < 16; ++i)
                  if (c0 + i < p.n_valid) dst[i] = v[i];
              }
            } else if (p.out_f32) {
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const int c = p.f32_coff + cb + i;
                if (c < p.n_valid) {
                  float x = v[i];
                  if (p.sigmoid) x = 1.f / (1.f + __expf(-x));
                  p.out_f32[(((size_t)img * p.n_valid + c) * p.Ho + oy) * p.Wo + ox] = x;
                }
              }
            }
            if constexpr (kSums) {
              if (p.sum_part) {
                if (j == 0) {
#pragma unroll
                  for (int i = 0; i < 16; ++i) sacc[i] += v[i];
                } else {
#pragma unroll
                  for (int i = 0; i < 16; ++i) sacc[16 + i] += v[i];
                }
              }
            }
            if (p.head_ko) {
#pragma unroll
              for (int k = 0; k < kMaxHeadOut; ++k) {
                if (k < p.head_ko) {
                  const float* w = s_head + k * BN + cb;
                  float a = hacc[k];
#pragma unroll
                  for (int i = 0; i < 16; ++i) a = fmaf(w[i], v[i], a);
                  hacc[k] = a;
                }
              }
            }
          }
        }
        if (p.head_ko) {
          // the two column halves of a pixel live in two warps of the same lane quarter: the upper half hands its
          // partial dot products over through shared memory (named barrier of the 64 threads involved)
          if (half == 1) {
#pragma unroll
            for (int k = 0; k < kMaxHeadOut; ++k) if (k < p.head_ko) s_hx[k * 128 + r] = hacc[k];
          }
          ptx::bar_sync(1 + q, 64);
          if (half == 0 && valid) {
#pragma unroll
            for (int k = 0; k < kMaxHeadOut; ++k) {
              if (k < p.head_ko) {
                float x = hacc[k] + s_hx[k * 128 + r] + p.head_b[k];
                if (p.head_sigmoid_mask & (1 << k)) x = 1.f / (1.f + __expf(-x));
                p.head_out[k][(size_t)img * p.head_img_stride[k] + (size_t)oy * p.Wo + ox] = x;
              }
            }
          }
          ptx::bar_sync(1 + q, 64);
        }
      }
      ptx::bar_sync(5, kEpiWarps * 32);        // every warp has read the accumulator tile before the next tile overwrites it
    }
    if (kSums && p.sum_part && sum_img >= 0) flush_sums(sum_img);
  }
}

// col_sums[img][c] = sum over the (CTA, lane quarter) partial rows, in a fixed order: block (bn, 16) -- 16 slices of the
// partial rows, independent loads issued in batches, then a fixed-order sum of the slices through shared memory
__global__ void col_sum_reduce_kernel(const float* __restrict__ part, int n_part, int n_img, int bn,
                                      float* __restrict__ out) {
  __shared__ float sm[16][64];
  ptx::griddep_launch_dependents();
  ptx::griddep_wait();                      // the partial rows come from the convolution just before
  const int img = blockIdx.x, c = threadIdx.x, sl = threadIdx.y;
  const int per = (n_part + 15) / 16;
  const int k0 = sl * per, k1 = min(n_part, k0 + per);
  float a = 0.f;
  for (int kb = k0; kb < k1; kb += 8) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = kb + i < k1 ? part[((size_t)(kb + i) * n_img + img) * bn + c] : 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) a += v[i];
  }
  sm[sl][c] = a;
  __syncthreads();
  if (sl == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) t += sm[i][c];
    out[(size_t)img * bn + c] = t;
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(ptr);
  }
  return fn;
}

int launch_col_sum_reduce(const float* part, int n_part, int n_img, float* out, cudaStream_t stream) {
  STP3_CUDA_OK(launch_pdl(col_sum_reduce_kernel, dim3(n_img), dim3(64, 16), 0, stream, part, n_part, n_img, 64, out));
  return STP3_OK;
}

}  // namespace stp3

using namespace stp3;

static int conv_num_sms() {
  static const int n = [] {
    int dev = 0, v = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();
  return n;
}

extern "C" size_t stp3_conv_col_sums_scratch_bytes(int n_img, int bn) {
  return (size_t)conv_num_sms() * 4 * (size_t)(n_img > 0 ? n_img : 0) * (size_t)(bn > 0 ? bn : 0) * sizeof(float);
}

extern "C" int stp3_conv_fwd(const stp3_conv_desc* d, const void* x_hi, const void* x_lo, const void* w,
                             const float* bias, const float* img_bias, const void* res_hi, const void* res_lo,
                             void* y_hi, void* y_lo, float* y_f32, const stp3_conv_head* head, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STP3_CHECK_ARG(d && x_hi && x_lo && w && bias, "stp3_conv_fwd: null pointer argument");
  STP3_CHECK_ARG((y_hi && y_lo) || y_f32 || head, "stp3_conv_fwd: no output tensor");
  if (head) {
    STP3_CHECK_ARG(head->n_out >= 1 && head->n_out <= kMaxHeadOut && head->w && head->b, "bad fused head");
    STP3_CHECK_ARG(d->bn <= 128, "a fused head needs bn <= 128");
    for (int k = 0; k < head->n_out; ++k) STP3_CHECK_ARG(head->out[k] != nullptr, "fused head: null output plane");
  }
  STP3_CHECK_ARG(d->B > 0 && d->T > 0 && d->H > 0 && d->W > 0 && d->Ho > 0 && d->Wo > 0, "non-positive dimension");
  const int T_total = d->T_total > 0 ? d->T_total : d->T;
  STP3_CHECK_ARG(d->t0 >= 0 && d->t0 + d->T <= T_total, "frame window [t0, t0+T) outside the input tensor");
  const int n_store = d->n_store > 0 ? d->n_store : d->bn;
  STP3_CHECK_ARG(n_store % 8 == 0 && n_store <= d->bn, "n_store must be a multiple of 8 and <= bn");
  STP3_CHECK_ARG(d->in_cstride % 64 == 0 && d->cin % 64 == 0 && d->cin_off % 64 == 0 && d->cin > 0 &&
                 d->cin_off + d->cin <= d->in_cstride, "input channels must be padded to multiples of 64");
  STP3_CHECK_ARG(d->bn == 64 || d->bn == 128 || d->bn == 256, "bn (padded output channels) must be 64, 128 or 256");
  STP3_CHECK_ARG(d->stride == 1 || d->stride == 2, "stride must be 1 or 2");
  STP3_CHECK_ARG(d->ntaps >= 1 && d->ntaps <= kMaxTaps, "ntaps out of range");
  if (y_hi) STP3_CHECK_ARG(d->out_cstride % 8 == 0 && d->out_coff % 8 == 0 && d->out_coff + n_store <= d->out_cstride,
                           "output channel window does not fit the output tensor");
  if (d->res_mode) STP3_CHECK_ARG(res_hi && res_lo && d->res_cstride % 8 == 0 && d->res_coff % 8 == 0 &&
                                  d->res_coff + d->bn <= d->res_cstride, "bad residual tensor");
  if (y_f32) STP3_CHECK_ARG(d->n_valid > 0 && d->n_valid <= d->bn, "n_valid out of range");
  PFN_tmapEncodeTiled enc = encode_fn();
  if (!enc) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");

  // tuning knobs (0 = automatic): desc->tune_group, or the STP3_CONV_GROUP environment variable.  tune_n_sub is
  // accepted for ABI compatibility; the tile is always 8 x 16 pixels.
  static const int env_group = [] { const char* e = getenv("STP3_CONV_GROUP"); return e ? atoi(e) : 0; }();
  const int want_group_raw = d->tune_group ? d->tune_group : env_group;
  const int want_group = want_group_raw & 3;
  static const bool use_pdl = stp3_pdl_enabled("STP3_CONV_PDL");
  const bool stream_weights = (want_group_raw & 4) != 0;    // +4: keep the weights in the ring even if they would fit
  // +8: stacked [W_hi; W_lo] operand (bn = 64 only).  Untuned (tune_group == 0) multi-tap 64-column layers use it: it
  // reads the activation tile twice instead of three times
  const bool stack = d->bn == 64 && ((want_group_raw & 8) != 0 || (want_group_raw == 0 && d->ntaps > 1));
  // taps that can share one activation load: runs (<= 4) of consecutive taps with the same (dt, dx) and dy advancing
  // by the stride
  ConvParams p;
  p.n_groups = 0; p.gmax = 1;
  for (int i = 0; i < d->ntaps;) {
    int g = 1;
    if (want_group != 1)
      while (g < 4 && i + g < d->ntaps && d->taps[i + g][0] == d->taps[i][0] && d->taps[i + g][2] == d->taps[i][2] &&
             d->taps[i + g][1] == d->taps[i][1] + g * d->stride)
        ++g;
    p.gstart[p.n_groups] = (unsigned char)i; p.gsize[p.n_groups] = (unsigned char)g; ++p.n_groups;
    if (g > p.gmax) p.gmax = g;
    i += g;
  }
  const int group = p.gmax;
  const int tile_h = kSubH;
  const int box_h = kSubH + (group - 1);                                 // image rows one CTA loads per stage

  CUtensorMap tm_hi, tm_lo, tm_w;
  {
    const cuuint64_t dims[5] = {(cuuint64_t)d->in_cstride, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)T_total,
                                (cuuint64_t)d->B};
    const cuuint64_t strides[4] = {(cuuint64_t)d->in_cstride * 2, (cuuint64_t)d->W * d->in_cstride * 2,
                                   (cuuint64_t)d->H * d->W * d->in_cstride * 2,
                                   (cuuint64_t)T_total * d->H * d->W * d->in_cstride * 2};
    const cuuint32_t box[5] = {(cuuint32_t)kBK, (cuuint32_t)((kTileW - 1) * d->stride + 1),
                               (cuuint32_t)((box_h - 1) * d->stride + 1), 1, 1};
    const cuuint32_t estr[5] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1, 1};
    CUresult r1 = enc(&tm_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x_hi), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CUresult r2 = enc(&tm_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x_lo), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
      return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation) failed: %d %d", (int)r1, (int)r2);
  }
  const int kblocks = d->cin / kBK;
  const int bn_launch = d->bn == 256 ? 128 : d->bn;     // 256 output channels run as two 128-column launches
  // the MMAs cover only the columns that carry weights (n_cols, rounded up to a multiple of 16)
  const int n_mma = d->bn <= 128 && d->n_cols > 0 && d->n_cols < d->bn ? ((d->n_cols + 15) / 16) * 16 : bn_launch;
  {
    const cuuint64_t dims[2] = {(cuuint64_t)kBK, (cuuint64_t)d->ntaps * kblocks * 2 * d->bn};
    const cuuint64_t strides[1] = {(cuuint64_t)kBK * 2};
    const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)n_mma};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  }

  p.n_img = d->B * d->T; p.T = d->T; p.t0 = d->t0; p.Ho = d->Ho; p.Wo = d->Wo;
  p.T_total = T_total;
  p.H = d->H; p.W = d->W;
  p.skip_t = 0;                                     // safe only if some tap always stays inside: the centre tap
  for (int i = 0; i < d->ntaps; ++i) if (d->taps[i][0] == 0 && d->taps[i][1] == 0 && d->taps[i][2] == 0) p.skip_t = 1;
  p.tiles_x = ceil_div(d->Wo, kTileW); p.tiles_y = ceil_div(d->Ho, tile_h);
  p.stride = d->stride; p.kblocks = kblocks; p.cin_off = d->cin_off; p.ntaps = d->ntaps;
  {
    const int k_lo = d->k_hi > 0 ? d->k_lo : 0, k_hi = d->k_hi > 0 ? d->k_hi : d->cin;
    STP3_CHECK_ARG(k_lo % 16 == 0 && k_hi % 16 == 0 && k_lo >= 0 && k_lo < k_hi && k_hi <= d->cin &&
                   k_lo < kBK && k_hi > d->cin - kBK, "k_lo / k_hi: multiples of 16 inside the first / last 64-channel block");
    p.ks_first = k_lo / 16;
    p.ks_end = (k_hi - (kblocks - 1) * kBK) / 16;
    STP3_CHECK_ARG(kblocks > 1 || p.ks_first < p.ks_end, "empty K range");
  }
  p.a_plane_bytes = box_h * kTileW * kBK * 2; p.w_rows = d->bn; p.n_mma = n_mma;
  for (int i = 0; i < d->ntaps; ++i) { p.tap[i][0] = d->taps[i][0]; p.tap[i][1] = d->taps[i][1]; p.tap[i][2] = d->taps[i][2]; p.tap[i][3] = 0; }
  p.relu = d->relu; p.res_mode = d->res_mode;
  p.res_hi = static_cast<const __nv_bfloat16*>(res_hi); p.res_lo = static_cast<const __nv_bfloat16*>(res_lo);
  p.res_cstride = d->res_cstride;
  p.out_hi = static_cast<__nv_bfloat16*>(y_hi); p.out_lo = static_cast<__nv_bfloat16*>(y_lo);
  p.out_cstride = d->out_cstride;
  p.out2_hi = static_cast<__nv_bfloat16*>(d->y2_hi); p.out2_lo = static_cast<__nv_bfloat16*>(d->y2_lo);
  p.out2_cstride = d->out2_cstride; p.out2_coff = d->out2_coff; p.relu2 = d->relu2;
  p.n_store2 = d->n_store2 > 0 ? d->n_store2 : 64;
  if (d->y2_hi) {
    STP3_CHECK_ARG(d->bn == 128 && d->y2_lo && y_hi && !d->res_mode && !head && !y_f32 && !d->col_sums,
                   "second destination: 128-column convolutions with plain hi/lo outputs only");
    STP3_CHECK_ARG(n_store <= 64 && p.n_store2 % 8 == 0 && p.n_store2 <= 64 && d->out2_cstride % 8 == 0 &&
                   d->out2_coff % 8 == 0 && d->out2_coff + p.n_store2 <= d->out2_cstride,
                   "second destination: channel window does not fit");
  }
  p.out_f32 = y_f32; p.n_valid = d->n_valid; p.sigmoid = d->sigmoid;
  p.f32_nhwc = d->f32_layout;
  STP3_CHECK_ARG(d->f32_layout == 0 || d->f32_layout == 1, "f32_layout must be 0 (n_img, n_valid, Ho, Wo) or 1 (n_img, Ho, Wo, n_valid)");
  if (y_f32 && d->f32_layout == 1)
    STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(y_f32) & 31) == 0 && !d->sigmoid,
                   "channels-last y_f32 must be 32-byte aligned (and carries no sigmoid)");
  p.img_bias_stride = d->bn;
  p.head_ko = 0; p.head_w = nullptr; p.head_b = nullptr; p.head_sigmoid_mask = 0;
  for (int k = 0; k < kMaxHeadOut; ++k) { p.head_out[k] = nullptr; p.head_img_stride[k] = 0; }
  if (head) {
    p.head_ko = head->n_out; p.head_w = head->w; p.head_b = head->b; p.head_sigmoid_mask = head->sigmoid_mask;
    for (int k = 0; k < head->n_out; ++k) { p.head_out[k] = head->out[k]; p.head_img_stride[k] = head->img_stride[k]; }
  }
  const int k_iters = d->ntaps * kblocks;
  const bool full_k = p.ks_first == 0 && p.ks_end == kBK / 16;
  const long long nblk = (long long)p.n_img * p.tiles_x * p.tiles_y;
  STP3_CHECK_ARG(nblk > 0 && nblk < (1ll << 31), "grid too large");
  p.n_tiles = (int)nblk;
  const int num_sms = conv_num_sms();
  unsigned grid = (unsigned)(nblk < num_sms ? nblk : num_sms);           // persistent: one CTA per SM
  const size_t smem_cap = 227 * 1024;
  const size_t a_stage = 2 * (size_t)p.a_plane_bytes;

  int launched_grid = (int)grid;
  p.sum_part = nullptr;
  if (d->col_sums) {
    STP3_CHECK_ARG(d->bn == 64, "col_sums: 64-column convolutions only");
    STP3_CHECK_ARG(d->col_sums_scratch && d->col_sums_scratch_bytes >= stp3_conv_col_sums_scratch_bytes(p.n_img, 64),
                   "col_sums: scratch buffer missing or smaller than stp3_conv_col_sums_scratch_bytes()");
    p.sum_part = static_cast<float*>(d->col_sums_scratch);
    // CTAs that never see an image leave its partial rows untouched: start from zeros
    STP3_CUDA_OK(cudaMemsetAsync(p.sum_part, 0, (size_t)grid * 4 * p.n_img * 64 * sizeof(float), stream));
  }

  for (int part = 0; part * bn_launch < d->bn; ++part) {
    const int coff = part * bn_launch;
    p.w_row_off = coff;
    p.bias = bias + coff;
    p.img_bias = img_bias ? img_bias + coff : nullptr;
    p.res_coff = d->res_coff + coff;
    p.out_coff = d->out_coff + coff;
    p.n_store = n_store - coff < bn_launch ? (n_store - coff > 0 ? n_store - coff : 0) : bn_launch;
    p.f32_coff = coff;
    auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
    p.vec256 = (y_hi && d->out_cstride % 16 == 0 && p.out_coff % 16 == 0 && al32(y_hi) && al32(y_lo) ? 1 : 0) |
               (d->res_mode && d->res_cstride % 16 == 0 && p.res_coff % 16 == 0 && al32(res_hi) && al32(res_lo) ? 2 : 0) |
               (d->y2_hi && d->out2_cstride % 16 == 0 && d->out2_coff % 16 == 0 && al32(d->y2_hi) && al32(d->y2_lo) ? 4 : 0);
#define STP3_LAUNCH_CONV(BN_, STACK_, FULLK_)                                                                     \
    do {                                                                                                          \
      using SM = ConvSmem<BN_, STACK_>;                                                                           \
      p.b_rows = FULLK_ ? BN_ : n_mma;                                                                            \
      p.b_tile_bytes = 2 * p.b_rows * kBK * 2;                                                                    \
      p.b_load_bytes = 2 * n_mma * kBK * 2;                                                                       \
      const size_t avail = smem_cap - 1024 - SM::tail_bytes();                                                    \
      const size_t wbytes = (size_t)k_iters * (size_t)p.b_tile_bytes;                                             \
      /* small weight tensors stay resident in smem next to >= 2 activation stages */                            \
      const bool res = !stream_weights && wbytes + 2 * a_stage <= avail;                                          \
      int na, nb;                                                                                                 \
      if (res) {                                                                                                  \
        na = (int)((avail - wbytes) / a_stage); nb = 0;                                                           \
      } else {                                                                                                    \
        /* as many activation stages as fit beside two weight slots, then fill up with weight slots (a slot is  */ \
        /* released one wgmma group after its last reader, so two slots keep a tap group of any size moving)    */ \
        na = (int)((avail - 2 * (size_t)p.b_tile_bytes) / a_stage);                                               \
        if (na > kMaxAStages) na = kMaxAStages;                                                                   \
        if (na < 2 || (size_t)na * a_stage + 2 * (size_t)p.b_tile_bytes > avail)                                  \
          return set_error(STP3_EUNSUPPORTED, "convolution does not fit in shared memory");                       \
        nb = (int)((avail - (size_t)na * a_stage) / (size_t)p.b_tile_bytes);                                      \
      }                                                                                                           \
      if (na > kMaxAStages) na = kMaxAStages;                                                                     \
      if (nb > kMaxBStages) nb = kMaxBStages;                                                                     \
      p.na_stages = na; p.nb_stages = nb; p.b_resident = res ? 1 : 0;                                             \
      const size_t smem_bytes = 1024 + na * a_stage + (res ? wbytes : (size_t)nb * (size_t)p.b_tile_bytes) + SM::tail_bytes(); \
      auto kern = conv_igemm_kernel<BN_, STACK_, FULLK_>;                                                         \
      /* once per kernel instantiation and device: the attribute call costs microseconds on every eager launch */ \
      static thread_local int attr_dev = -1;                                                                      \
      int cur_dev = 0; cudaGetDevice(&cur_dev);                                                                   \
      if (attr_dev != cur_dev) {                                                                                  \
        STP3_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap));     \
        attr_dev = cur_dev;                                                                                       \
      }                                                                                                           \
      cudaLaunchConfig_t cfg = {};                                                                                \
      cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kConvThreads);                                                \
      cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;                                                     \
      cudaLaunchAttribute attr[1];                                                                                \
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                            \
      attr[0].val.programmaticStreamSerializationAllowed = 1;                                                     \
      cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;                                                           \
      launched_grid = (int)cfg.gridDim.x;                                                                         \
      STP3_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tm_hi, tm_lo, tm_w, p));                                        \
    } while (0)
    if (bn_launch == 64) {
      if (stack) { if (full_k) STP3_LAUNCH_CONV(64, true, true); else STP3_LAUNCH_CONV(64, true, false); }
      else { if (full_k) STP3_LAUNCH_CONV(64, false, true); else STP3_LAUNCH_CONV(64, false, false); }
    } else {
      if (full_k) STP3_LAUNCH_CONV(128, false, true); else STP3_LAUNCH_CONV(128, false, false);
    }
#undef STP3_LAUNCH_CONV
    STP3_CUDA_OK(cudaGetLastError());
  }
  if (p.sum_part) {
    STP3_CUDA_OK(launch_pdl(col_sum_reduce_kernel, dim3(p.n_img), dim3(64, 16), 0, stream, (const float*)p.sum_part,
                            launched_grid * 4, p.n_img, 64, static_cast<float*>(d->col_sums)));
  }
  return STP3_OK;
}
