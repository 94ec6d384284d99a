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
//   item     : 128 output pixels (8 x 16 of one image) x one block of BN output channels (64 / 128).  A convolution
//              wider than its column block (256 columns, or 128 / 256 in 64-column blocks) is still ONE launch: the
//              blocks of a pixel tile are consecutive work items, so the tile's activation windows stay hot in L2
//   K loop   : taps x (Cin / 64); TMA brings A_hi, A_lo (128 or 160 pixel rows x 64 bf16, 128B-swizzled; one load
//              serves the three dy taps of a 3x3) and B_hi, B_lo (BN x 64; small weight tensors stay resident in
//              smem) through separate rings; each warpgroup issues 4 (K = 16) x 3 wgmma per tap for its 64 rows
//   CTA      : persistent, one per SM, walks items blockIdx.x + i*gridDim.x
//   warps    : 0..7 = two MMA warpgroups (rows 0..63 / 64..127 of the tile): wgmma only, then their fragments into
//              the shared accumulator tile; 8..15 = two epilogue warpgroups (shared accumulator tile -> global) that
//              drain tile u while the MMA warpgroups multiply tile u+1; 16 = TMA producer (17..19 leave at once)
//
// Reference layers: stp3/layers/temporal.py:252-489, stp3/layers/convolutions.py:183-280, stp3/models/decoder.py.
#include <cuda_bf16.h>

#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "pipeline.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kMmaWarps = 8;                     // two warpgroups, 64 accumulator rows each
constexpr int kEpiWarps = 8;                     // two warps per 32-row quarter of the tile, each owning half of the columns
constexpr int kProducerWarp = kMmaWarps + kEpiWarps;
constexpr int kConvThreads = (kProducerWarp + 4) * 32;   // the producer has a warpgroup of its own for setmaxnreg
// per-thread registers of each role (setmaxnreg): the MMA warpgroups hold the accumulator (64 registers for BN = 128
// and for the stacked BN = 64), the epilogue its chunk, residual, column-sum and head arrays.  ptxas -v reports no
// spills in any instantiation with this split.  setmaxnreg.inc only takes registers that another warpgroup of the CTA
// gave back with setmaxnreg.dec: the five roles together must fit the CTA's launch allocation (96 per thread for 640
// threads), or an inc waits forever.
constexpr int kProducerRegs = 24, kMmaRegs = 96, kEpiRegs = 128;
constexpr int kLaunchRegs = 65536 / kConvThreads / 8 * 8;
static_assert(kProducerRegs + 2 * kMmaRegs + 2 * kEpiRegs <= 5 * kLaunchRegs, "setmaxnreg split exceeds the CTA's registers");
// the single shared accumulator tile is handed over with two named barriers of the MMA and epilogue threads (ids
// 1..4 are the epilogue's column-half pairs): "full" (MMA arrive, epilogue sync) and "free" (the reverse)
constexpr int kBarAccFull = 5, kBarAccFree = 6;
constexpr int kHandoverThreads = (kMmaWarps + kEpiWarps) * 32;
// the epilogue threads alone: every row of the staging tile is written, its TMA stores may start
constexpr int kBarEpi = 7;
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kSubH = 8, kTileW = 16;           // one tile = 8 x 16 pixels = 128 accumulator rows
constexpr int kBK = 64;                         // channels per K step (one 128-byte swizzle row of bf16)
constexpr int kMaxTaps = 49;
constexpr int kMaxAStages = 4, kMaxBStages = 8;
constexpr int kMaxHeadOut = 8;
constexpr size_t kSmemCap = 227 * 1024;           // dynamic shared memory one CTA may ask for

struct ConvParams {
  int n_img, T, t0, Ho, Wo;
  int T_total;              // frames of the input tensor
  int H, W;                 // input image size
  int skip_t;               // skip tap groups whose window lies entirely in the zero padding for the whole tile (frame
                            // outside [0, T_total): causal convs at t = 0; rows / columns outside the image: dilated convs)
  int tiles_x, tiles_y, n_tiles;
  int n_nblk;               // column blocks of BN output channels per pixel tile; work item i = (tile i / n_nblk, block
                            // i % n_nblk).  Block nb owns columns [nb * BN, nb * BN + BN) of the weights, the bias, the
                            // residual and every output
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
  signed char tap[kMaxTaps][4];   // (dt, dy, dx): input coordinate = output coordinate * stride + d
  const float* bias;        // [n_nblk * BN]
  const float* img_bias;    // [n_img][img_bias_stride] or null (replaces bias)
  int img_bias_stride;
  int relu;
  int res_mode;             // 0 none, 1 residual added before the activation, 2 after
  const __nv_bfloat16* res_hi;
  const __nv_bfloat16* res_lo;
  int res_cstride, res_coff;
  // hi/lo destinations (channels-last (n_img, Ho, Wo, cstride)) are written through the kernel's output tensor maps,
  // which start at the destination's channel offset and end after its n_store channels
  int out_hl;               // 0: no hi/lo output (out_f32 or a fused head only)
  int n_store;              // channels of the primary destination
  int vec256;               // bit 1: residual rows / windows are 32-byte aligned (256-bit loads)
  float* out_f32;           // optional (n_img, n_valid, Ho, Wo) fp32, the reference's NCHW layout
  int n_valid;
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
  int out2, relu2;
  // per-image column sums of the activated output (the consumer's pooling branches need sum over H*W): every epilogue
  // warp keeps running sums of its pixels in registers and writes one partial row per (CTA, row quarter, image) --
  // plain stores, fixed order: deterministic.  BN = 64 only.  sum_part: [gridDim.x][4][n_img][BN], zeroed by the host.
  float* sum_part;
  int swish;                // swish instead of ReLU on the primary destination (EfficientNet expand convolutions)
  long long w_img_rows;     // > 0: per-image weights, image i's blocks start w_img_rows rows further (streamed only)
};

// STACK (BN = 64 only): the hi and lo weight planes of a K step form ONE B operand of 2*BN rows, so a product is two
// MMAs instead of three -- A_hi x [W_hi; W_lo] (N = 2*BN) and A_lo x W_hi (N = BN) -- and the activation tile is read
// from shared memory twice instead of three times.  The register accumulator has 2*BN columns; the MMA warpgroups add
// columns c and b_rows + c on their way to the shared accumulator tile, which has BN columns either way.
template <int BN>
struct ConvSmem {
  // the tail behind the operand rings (or the resident weights), byte offsets from its start
  static constexpr int bias = 0;                                       // fp32 [n_nblk * BN]: the blocks beyond the first
                                                                       // lie over the head weights (n_nblk > 1: no head)
  static constexpr int head = bias + BN * 4;                           // fp32 [kMaxHeadOut][BN] fused head weights
  static constexpr int hx = head + kMaxHeadOut * BN * 4;               // fp32 [kMaxHeadOut][128] head partials handed between column halves
  static constexpr int wb = hx + kMaxHeadOut * 128 * 4;                // fp32 [kEpiWarps][64] per-image bias slice of each epilogue warp
  // fp32 [128][BN] accumulator tile, which the epilogue turns into the staging tile of the hi/lo output stores in
  // place: [BN / 64 channel planes][hi, lo part][128 pixels][64 bf16], each part 128-byte swizzled like the TMA loads
  // (1024-byte aligned: the tail starts on a 1024-byte boundary)
  static constexpr int acc = (wb + kEpiWarps * 64 * 4 + 1023) / 1024 * 1024;
  static constexpr int kStagePart = 128 * 128;                         // bytes of one (plane, part)
  static constexpr int bars = acc + BN / 64 * 2 * kStagePart;          // A ring, B ring, resident-weights barrier
  // Byte offset of accumulator (row, col).  Of the 16 columns of a chunk (col / 16), columns 0..7 lie in the hi part
  // and 8..15 in the lo part, each 8 in the two 16-byte slots of the row that the chunk's 8 hi (lo) bf16 outputs take
  // (slot s of row r at s ^ (r % 8)): the epilogue thread of a row overwrites exactly the accumulators it has read.
  static __device__ __forceinline__ int acc_off(int row, int col) {
    const int k = col & 15;
    const int slot = ((col & 63) >> 4) * 2 + ((k >> 2) & 1);
    return ((col >> 6) * 2 + (k >> 3)) * kStagePart + row * 128 + ((slot ^ (row & 7)) << 4) + (k & 3) * 4;
  }
  static constexpr size_t tail_bytes() { return bars + (2 * kMaxAStages + 2 * kMaxBStages + 8) * 8; }
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

// Persistent, warp-specialised implicit-GEMM convolution.
//   * A CTA walks work items blockIdx.x + i*gridDim.x: (pixel tile, column block) pairs, the blocks of a tile next to
//     each other.  A tile is 8x16 pixels = 128 accumulator rows, 64 per warpgroup.
//   * Activations and weights travel through separate shared-memory rings filled by one producer warp.  For 3x3 /
//     stride 1 / dilation 1 kernels one activation load of 10 image rows serves the three dy taps: their A operands are
//     the same smem tile at row offsets 0, 16, 32 (2 KB steps keep the 1024-byte swizzle alignment).
//   * wgmma groups are committed per tap; a ring slot is released once the group after the one that read it has been
//     issued and the reading group has retired (wgmma.wait_group 1), so the tensor pipe always has the next tap queued.
//   * At the end of a tile the MMA warpgroups wait until the epilogue has released the shared [128 rows][columns] fp32
//     accumulator tile, write their accumulators into it and go on with the next tile; the epilogue warpgroups give
//     every thread one pixel (row) and half of the columns.
// FULLK: every K = 16 step of every K block carries data (ks_first == 0, ks_end == 4).  Then a tap is a branch-free run
// of wgmma with N fixed at compile time (BN, 2 * BN for the stacked operand), which ptxas pipelines; any branch around
// the MMAs (skipped K steps, an N chosen at run time) makes it serialise them.
// OP: operand kind.  0 = bf16 hi/lo planes, three MMAs per product (fp32-equivalent); 1 = one bf16 plane, 2 = one fp16
// plane (autocast training): the activation stage and the weight tile hold one plane and each K step is one MMA.
template <int BN, bool STACK, bool FULLK, int OP = 0>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_o_hi,
                  const __grid_constant__ CUtensorMap tm_o_lo, const __grid_constant__ CUtensorMap tm_o2_hi,
                  const __grid_constant__ CUtensorMap tm_o2_lo, const ConvParams p) {
  using S = ConvSmem<BN>;
  static_assert(!STACK || BN == 64, "stacked weight operand: BN = 64 only");
  static_assert(OP == 0 || !STACK, "one-plane operands: no stacked weight operand");
  constexpr int kPlanes = OP == 0 ? 2 : 1;             // planes per activation stage and per weight tile
  constexpr int kAccRegs = (STACK ? 2 * BN : BN) / 2;   // accumulator registers per thread (64 rows x columns per warpgroup)
  const int kBRows = p.b_rows;
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte alignment for the 128-byte swizzle; plain offset arithmetic keeps the pointer in the shared state space
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int k_iters = p.ntaps * p.kblocks;
  const bool resident = p.b_resident != 0;
  const int a_stage_bytes = kPlanes * p.a_plane_bytes;
  unsigned char* a_ring = smem;
  unsigned char* b_ring = a_ring + (size_t)p.na_stages * a_stage_bytes;            // ring, or the resident weights
  unsigned char* tail = b_ring + (size_t)(resident ? k_iters : p.nb_stages) * p.b_tile_bytes;
  float* s_bias = reinterpret_cast<float*>(tail + S::bias);
  float* s_head = reinterpret_cast<float*>(tail + S::head);
  float* s_hx = reinterpret_cast<float*>(tail + S::hx);
  float* s_wb = reinterpret_cast<float*>(tail + S::wb);
  unsigned char* s_acc = tail + S::acc;
  uint64_t* bars = reinterpret_cast<uint64_t*>(tail + S::bars);
  Ring ra{bars, bars + kMaxAStages, p.na_stages};
  Ring rb{bars + 2 * kMaxAStages, bars + 2 * kMaxAStages + kMaxBStages, p.nb_stages};   // no slots: resident weights
  uint64_t* bres_bar = bars + 2 * (kMaxAStages + kMaxBStages);
  // The MMA warpgroups walk both rings with counters of their own: the same walk through a Ring makes ptxas spill more
  // in four of the six instantiations
  uint64_t* const a_full = ra.full;
  uint64_t* const a_empty = ra.empty;
  uint64_t* const b_full = rb.full;
  uint64_t* const b_empty = rb.empty;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // Programmatic dependent launch: the next conv of the stream may set up (barriers, resident weights) on SMs this grid
  // has left; this grid's own set-up ran while its predecessor drained.  Only module constants (bias, weights, head
  // weights) are read before griddep_wait().
  ptx::griddep_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    ptx::prefetch_tmap(&tm_a_hi); if constexpr (OP == 0) ptx::prefetch_tmap(&tm_a_lo); ptx::prefetch_tmap(&tm_w);
    if (p.out_hl) { ptx::prefetch_tmap(&tm_o_hi); ptx::prefetch_tmap(&tm_o_lo); }
    if (p.out2) { ptx::prefetch_tmap(&tm_o2_hi); ptx::prefetch_tmap(&tm_o2_lo); }
    ra.init(2); rb.init(2);
    ptx::mbar_init(bres_bar, 1);
    ptx::fence_mbar_init();
  }
  static_assert(kMaxHeadOut * BN >= 256 - BN, "the bias of every column block fits in the bias and head-weight areas");
  for (int i = threadIdx.x; i < p.n_nblk * BN; i += blockDim.x) s_bias[i] = p.bias[i];
  for (int i = threadIdx.x; i < p.head_ko * BN; i += blockDim.x) s_head[i] = p.head_w[i];
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int n_groups = p.n_groups;
  const int tile_h = kSubH;
  const int n_items = p.n_tiles * p.n_nblk;

  if (warp >= kProducerWarp) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp != kProducerWarp) return;
    // ===================== TMA producer (whole warp walks the loops; one elected lane issues) =====================
    // load_b: the weight tile of K step `it` into `dst` (called by the elected lane; transaction bytes on `bar`)
    auto load_b = [&](unsigned char* dst, int it, uint64_t* bar, int img_w, int nb) {
      const int row_hi = (int)((it * kPlanes) * p.w_rows + nb * BN + img_w * p.w_img_rows), row_lo = row_hi + p.w_rows;
      ptx::tma_load_2d(dst, &tm_w, bar, 0, row_hi);                       // [W_hi; W_lo], also the stacked operand
      if constexpr (OP == 0) ptx::tma_load_2d(dst + kBRows * kBK * 2, &tm_w, bar, 0, row_lo);
    };
    if (resident && ptx::elect_one_sync()) {
      ptx::mbar_arrive_expect_tx(bres_bar, (uint32_t)(k_iters * p.b_load_bytes));
      for (int it = 0; it < k_iters; ++it) load_b(b_ring + (size_t)it * p.b_tile_bytes, it, bres_bar, 0, 0);
    }
    __syncwarp();
    ptx::griddep_wait();                        // activations come from the preceding kernel
    for (int item = cta; item < n_items; item += n_cta) {
      const int tile = item / p.n_nblk, nb = item % p.n_nblk;
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
          ra.produce((uint32_t)a_stage_bytes, [&](int s, uint64_t* bar) {
            unsigned char* sa = a_ring + (size_t)s * a_stage_bytes;
            const int c = p.cin_off + kb * kBK;
            ptx::tma_load_5d(sa, &tm_a_hi, bar, c, x, y, t, bidx);
            if constexpr (OP == 0) ptx::tma_load_5d(sa + p.a_plane_bytes, &tm_a_lo, bar, c, x, y, t, bidx);
          });
          if (!resident) {
            for (int j = 0; j < gsz; ++j) {
              const int it = (tap0 + j) * p.kblocks + kb;          // [tap][kb][plane][rows] blocks of 64-wide rows
              rb.produce((uint32_t)p.b_load_bytes,
                         [&](int s, uint64_t* bar) { load_b(b_ring + (size_t)s * p.b_tile_bytes, it, bar, img, nb); });
            }
          }
        }
      }
    }
  } else if (warp < kMmaWarps) {
    // ===================== two MMA warpgroups =====================
    ptx::setmaxnreg_inc<kMmaRegs>();
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
      PendingSlots pend{a_empty, b_empty, wg_leader};
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
                if constexpr (OP != 0) {
                  wg::mma_plane<OP, BN>(accr, da_hi + koff, db_hi + koff, acc0);
                } else if constexpr (STACK) {
                  wg::mma_bf16<2 * BN>(accr, da_hi + koff, db_hi + koff, acc0);                // A_hi x [W_hi; W_lo]
                  wg::mma_bf16<BN>(accr, da_lo + koff, db_lo + koff, 1);                       // A_lo x W_hi
                } else {
                  wg::mma_hilo<BN>(accr, da_hi + koff, da_lo + koff, db_hi + koff, db_lo + koff, acc0);
                }
              }
            } else {
#pragma unroll
              for (int k = 0; k < kBK / 16; ++k) {
                if (k < k_begin || k >= k_end) continue;               // K steps of pure channel padding
                const uint64_t koff = (uint64_t)((k * 16 * 2) >> 4);
                const uint32_t acc0 = accumulate | (uint32_t)(k > k_begin);
                if constexpr (OP != 0) {
                  wg::mma_plane_n<OP, BN>(p.n_mma, accr, da_hi + koff, db_hi + koff, acc0);
                } else if constexpr (STACK) {
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
            pend.release();
            pend.b = resident ? -1 : bs;
            if (j + 1 == gsz) pend.a = as;
            accumulate = 1;
            if (!resident) { if (++bs == p.nb_stages) { bs = 0; bph ^= 1; } }
          }
          if (++as == p.na_stages) { as = 0; aph ^= 1; }
        }
      }
      wg::wait<0>();
      pend.release();
      ptx::bar_sync(kBarAccFree, kHandoverThreads);      // the epilogue has read the previous tile's accumulators
      // registers -> s_acc (columns the MMAs computed).  Register i holds column 8 (i / 4) + 2 (lane % 4) + i % 2, so
      // the stacked operand's A_hi x W_lo partner of column c (column b_rows + c) is register i + kLo, kLo = b_rows / 2
      const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      auto to_smem = [&](auto lo) {
        constexpr int kLo = decltype(lo)::value;             // 0: not stacked
#pragma unroll
        for (int i = 0; i < (kLo ? kLo : kAccRegs); i += 2) {
          const int col = 8 * (i >> 2) + 2 * (lane & 3);
          if (kLo || col < kBRows) {
            const int row = row0 + 8 * ((i >> 1) & 1);
            float2 v = make_float2(accr[i], accr[i + 1]);
            if constexpr (kLo > 0) { v.x += accr[i + kLo]; v.y += accr[i + 1 + kLo]; }
            *reinterpret_cast<float2*>(s_acc + S::acc_off(row, col)) = v;
          }
        }
      };
      if constexpr (!STACK) {
        to_smem(std::integral_constant<int, 0>{});
      } else if constexpr (FULLK) {
        to_smem(std::integral_constant<int, BN / 2>{});
      } else {
        switch (kBRows) {                                     // n_mma: 16, 32, 48 or 64
          case 16: to_smem(std::integral_constant<int, 8>{}); break;
          case 32: to_smem(std::integral_constant<int, 16>{}); break;
          case 48: to_smem(std::integral_constant<int, 24>{}); break;
          default: to_smem(std::integral_constant<int, 32>{}); break;
        }
      }
      ptx::bar_arrive(kBarAccFull, kHandoverThreads);
    };
    for (int item = cta; item < n_items; item += n_cta) mma_tile(item / p.n_nblk);   // whichever column block: the producer chose the weights
  } else {
    // ===================== two epilogue warpgroups: shared accumulator tile -> registers -> global =====================
    ptx::setmaxnreg_inc<kEpiRegs>();
    const int e = warp - kMmaWarps;
    const int q = warp & 3;                      // 32-row quarter of the tile this warp drains
    const int half = e >> 2;                     // which half of the BN columns this warp handles
    constexpr int kColsPerWarp = BN / 2;
    const int col0 = half * kColsPerWarp;
    const int r = q * 32 + lane;                 // row of the tile = output pixel
    // activation of this warp's columns (the upper column half may belong to a second tensor)
    const bool second = BN == 128 && half == 1 && p.out2;
    const bool d_relu = (second ? p.relu2 : p.relu) != 0;
    const bool d_swish = !second && p.swish != 0;
    const bool store_hl = p.out_hl != 0;
    // the hi/lo outputs leave through the staging tile (the accumulator tile, overwritten chunk by chunk): one thread
    // stores the tile's box of each plane part with TMA (pixels outside the map and channels outside the destination's
    // window are clipped by the tensor maps) and waits until the stores have read the tile before it releases the
    // accumulator tile to the MMA warpgroups
    const bool store_issuer = e == 0 && lane == 0;
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
    for (int item = cta; item < n_items; item += n_cta) {
      // done with the previous item's accumulators (if any), and the TMA stores with its staging tile
      if (store_issuer) ptx::bulk_wait_read0();
      ptx::bar_arrive(kBarAccFree, kHandoverThreads);
      const int tile = item / p.n_nblk;
      const int cblk = (item % p.n_nblk) * BN;          // first column of this item's block in the whole convolution
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_t = (rem / p.tiles_x) * kSubH, ox = (rem % p.tiles_x) * kTileW + (r & 15);
      if (kSums && p.sum_part && img != sum_img) {      // tiles come in image order: hand the finished image over
        if (sum_img >= 0) flush_sums(sum_img);
        sum_img = img;
      }
      // latency hiding: the residual of the first chunk and this warp's slice of the per-image bias are requested
      // before waiting for the accumulator; every later residual chunk as soon as the previous one has been added
      uint32_t nh[8] = {}, nl[8] = {};          // stay zero for pixels outside the map
      auto request_residual = [&](int j) {
        const int oy = oy_t + (r >> 4);
        if (oy < p.Ho && ox < p.Wo) {
          const size_t off = (((size_t)img * p.Ho + oy) * p.Wo + ox) * p.res_cstride + p.res_coff + cblk + col0 + j * 16;
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
      const float* bsrc = s_bias + cblk;          // bias of the block's column c at bsrc[c]
      if (p.img_bias) {
        const float* ib = p.img_bias + (size_t)img * p.img_bias_stride + cblk + col0;
        float* wb = s_wb + e * 64;
        __syncwarp();                             // every lane is done with the previous tile's slice
#pragma unroll
        for (int i = lane; i < kColsPerWarp; i += 32) wb[i] = *(reinterpret_cast<const volatile float*>(ib) + i);
        __syncwarp();
        bsrc = wb - col0;
      }
      ptx::bar_sync(kBarAccFull, kHandoverThreads);     // the MMA warpgroups have written this tile's accumulators
      {
        const int oy = oy_t + (r >> 4);
        const bool valid = oy < p.Ho && ox < p.Wo;
        const size_t pix = ((size_t)img * p.Ho + oy) * p.Wo + ox;
        float hacc[kMaxHeadOut];
#pragma unroll
        for (int k = 0; k < kMaxHeadOut; ++k) hacc[k] = 0.f;
#pragma unroll 1
        for (int j = 0; j < kColsPerWarp / 16; ++j) {
          const int cb = col0 + j * 16;              // first column of this chunk in the block,
          const int cg = cblk + cb;                  // in the convolution
          // the chunk's four 16-byte slots of this row: hi part columns 0..3, 4..7, lo part columns 8..11, 12..15
          uint4* const s_hi0 = reinterpret_cast<uint4*>(s_acc + S::acc_off(r, cb));
          uint4* const s_hi1 = reinterpret_cast<uint4*>(s_acc + S::acc_off(r, cb + 4));
          uint4* const s_lo0 = reinterpret_cast<uint4*>(s_acc + S::acc_off(r, cb + 8));
          uint4* const s_lo1 = reinterpret_cast<uint4*>(s_acc + S::acc_off(r, cb + 12));
          uint32_t acc[16];
          const bool computed = cb < p.n_mma;        // columns beyond n_mma: zero weights, never multiplied
          if (computed) {
            const uint4 a0 = *s_hi0, a1 = *s_hi1, a2 = *s_lo0, a3 = *s_lo1;
            acc[0] = a0.x; acc[1] = a0.y; acc[2] = a0.z; acc[3] = a0.w;
            acc[4] = a1.x; acc[5] = a1.y; acc[6] = a1.z; acc[7] = a1.w;
            acc[8] = a2.x; acc[9] = a2.y; acc[10] = a2.z; acc[11] = a2.w;
            acc[12] = a3.x; acc[13] = a3.y; acc[14] = a3.z; acc[15] = a3.w;
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = 0u;
          }
          // every row, pixels outside the map too: the hi/lo stores clip them
          float v[16];
#pragma unroll
          for (int g = 0; g < 4; ++g) {            // bias: per-image slice (conv bias already folded in) or the conv's own
            const float4 b4 = *reinterpret_cast<const float4*>(bsrc + cb + 4 * g);
            v[4 * g + 0] = __uint_as_float(acc[4 * g + 0]) + b4.x;
            v[4 * g + 1] = __uint_as_float(acc[4 * g + 1]) + b4.y;
            v[4 * g + 2] = __uint_as_float(acc[4 * g + 2]) + b4.z;
            v[4 * g + 3] = __uint_as_float(acc[4 * g + 3]) + b4.w;
          }
          if (p.res_mode) {
#pragma unroll
            for (int e2 = 0; e2 < 8; ++e2) {
              const float2 r = ptx::join_hilo(nh[e2], nl[e2]);
              float& a0 = v[e2 * 2], &a1 = v[e2 * 2 + 1];
              if (p.res_mode == 1) { a0 += r.x; a1 += r.y; if (d_relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); } }
              else { if (d_relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); } a0 += r.x; a1 += r.y; }
            }
            // the next chunk's residual is in flight while this chunk is finished (one buffer of residual registers)
            if (j + 1 < kColsPerWarp / 16) request_residual(j + 1);
          } else if (d_relu) {
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
          }
          if (d_swish) {                           // after a res_mode 1 residual, like ReLU; swish launches take no res_mode 2
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = v[i] / (1.f + __expf(-v[i]));
          }
          if (store_hl) {
            uint32_t hw[8], lw[8];
#pragma unroll
            for (int e2 = 0; e2 < 8; ++e2) ptx::split_hilo(v[e2 * 2], v[e2 * 2 + 1], hw[e2], lw[e2]);
            *s_hi0 = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *s_hi1 = make_uint4(hw[4], hw[5], hw[6], hw[7]);
            *s_lo0 = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            *s_lo1 = make_uint4(lw[4], lw[5], lw[6], lw[7]);
          }
          if (valid) {
            if (p.out_f32 && p.f32_nhwc) {
              const int c0 = cg;
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
                const int c = cg + i;
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
        if (store_hl) {
          ptx::fence_proxy_async();                 // the generic-proxy writes are visible to the TMA stores
          ptx::bar_sync(kBarEpi, kEpiThreads);      // every row of the staging tile is written
          if (store_issuer) {
            const int ox0 = (rem % p.tiles_x) * kTileW;
#pragma unroll
            for (int pl = 0; pl < BN / 64; ++pl) {
              const uint32_t src = ptx::smem_u32(s_acc + pl * 2 * S::kStagePart);
              if (BN == 128 && pl == 1 && p.out2) {
                ptx::tma_store_4d(&tm_o2_hi, src, 0, ox0, oy_t, img);
                ptx::tma_store_4d(&tm_o2_lo, src + S::kStagePart, 0, ox0, oy_t, img);
              } else if (cblk + pl * 64 < p.n_store) {
                ptx::tma_store_4d(&tm_o_hi, src, cblk + pl * 64, ox0, oy_t, img);
                ptx::tma_store_4d(&tm_o_lo, src + S::kStagePart, cblk + pl * 64, ox0, oy_t, img);
              }
            }
            ptx::bulk_commit();
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
    }
    if (kSums && p.sum_part && sum_img >= 0) flush_sums(sum_img);
    if (store_issuer) ptx::bulk_wait0();            // the staging tile is read and the last tile's outputs are written
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
int launch_col_sum_reduce(const float* part, int n_part, int n_img, float* out, cudaStream_t stream) {
  STP3_CUDA_OK(launch_pdl(kPdlAux, col_sum_reduce_kernel, dim3(n_img), dim3(64, 16), 0, stream, part, n_part, n_img, 64, out));
  return STP3_OK;
}

template <int BN, bool STACK, bool FULLK, int OP = 0>
static int launch_conv(const ConvParams& p, const CUtensorMap& tm_hi, const CUtensorMap& tm_lo, const CUtensorMap& tm_w,
                       const CUtensorMap (&tm_o)[4], size_t smem_bytes, unsigned grid, cudaStream_t stream) {
  constexpr auto kern = conv_igemm_kernel<BN, STACK, FULLK, OP>;
  STP3_CUDA_OK(set_max_dynamic_smem<kern>((int)kSmemCap));
  STP3_CUDA_OK(launch_pdl(kPdlConv, kern, dim3(grid), dim3(kConvThreads), smem_bytes, stream, tm_hi, tm_lo, tm_w,
                          tm_o[0], tm_o[1], tm_o[2], tm_o[3], p));
  return STP3_OK;
}

// What the host decides from the descriptor alone: the instantiation, the work items and the ring depths.
// stp3_conv_fwd launches it, stp3_conv_tiling reports it.
struct ConvPlan {
  int bn_blk;               // column-block width = the kernel's BN
  bool stack, full_k;
  int box_h;                // image rows of one activation stage
  int k_iters;
  unsigned grid;
  size_t smem_bytes;
};

// Checks every rule of the descriptor that needs no tensor pointer and fills the geometry, tiling and ring fields of p.
// operand: STP3_OPERAND_* (one-plane operands halve the activation stage and the weight tile and never stack).
static int plan_conv(const stp3_conv_desc* d, bool has_head, int n_sm, ConvParams& p, ConvPlan& t, int operand = 0) {
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
  STP3_CHECK_ARG(!d->swish || (!d->relu && d->res_mode != 2 && !d->y2_hi), "swish: not with relu, res_mode 2 or a second destination");
  if (d->w_img_stride)
    STP3_CHECK_ARG(d->w_img_stride > 0 && d->w_img_stride % 64 == 0 &&
                   d->w_img_stride >= (long long)d->ntaps * (d->cin / 64) * 2 * d->bn * 64,
                   "w_img_stride: a multiple of 64 elements, at least one image's weight blocks");
  STP3_CHECK_ARG(d->f32_layout == 0 || d->f32_layout == 1, "f32_layout must be 0 (n_img, n_valid, Ho, Wo) or 1 (n_img, Ho, Wo, n_valid)");

  // column blocks: tune_bn, or as wide as the kernel goes (128)
  STP3_CHECK_ARG(d->tune_bn == 0 || ((d->tune_bn == 64 || d->tune_bn == 128) && d->tune_bn <= d->bn),
                 "tune_bn (column-block width) must be 0, 64 or 128 and <= bn");
  t.bn_blk = d->tune_bn ? d->tune_bn : (d->bn == 256 ? 128 : d->bn);
  p.n_nblk = d->bn / t.bn_blk;
  STP3_CHECK_ARG(p.n_nblk == 1 || (!has_head && !d->y2_hi && !d->col_sums),
                 "a fused head, a second destination and col_sums need the convolution's columns in one block (tune_bn)");

  // tuning knobs (0 = automatic): desc->tune_group, or the STP3_CONV_GROUP environment variable.  tune_n_sub is
  // accepted for ABI compatibility; the tile is always 8 x 16 pixels.
  static const int env_group = [] { const char* e = getenv("STP3_CONV_GROUP"); return e ? atoi(e) : 0; }();
  const int want_group_raw = d->tune_group ? d->tune_group : env_group;
  const int want_group = want_group_raw & 3;
  // +4: keep the weights in the ring even if they would fit; per-image weights always stream, and so do the weights
  // of several column blocks (a CTA meets all of them)
  const bool stream_weights = (want_group_raw & 4) != 0 || d->w_img_stride != 0 || p.n_nblk > 1;
  // +8: stacked [W_hi; W_lo] operand (64-column blocks only).  Untuned (tune_group == 0) multi-tap layers in 64-column
  // blocks use it: it reads the activation tile twice instead of three times
  t.stack = operand == 0 && t.bn_blk == 64 && ((want_group_raw & 8) != 0 || (want_group_raw == 0 && d->ntaps > 1));
  // taps that can share one activation load: runs (<= 4) of consecutive taps with the same (dt, dx) and dy advancing
  // by the stride
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
  t.box_h = kSubH + (p.gmax - 1);                                        // image rows one CTA loads per stage

  const int kblocks = d->cin / kBK;
  // the MMAs cover only the columns that carry weights (n_cols, rounded up to a multiple of 16); with several column
  // blocks every block runs at full width (the padding rows are zeros)
  const int n_mma = p.n_nblk == 1 && d->n_cols > 0 && d->n_cols < d->bn ? ((d->n_cols + 15) / 16) * 16 : t.bn_blk;
  p.n_img = d->B * d->T; p.T = d->T; p.t0 = d->t0; p.Ho = d->Ho; p.Wo = d->Wo;
  p.T_total = T_total;
  p.H = d->H; p.W = d->W;
  p.skip_t = 0;                                     // safe only if some tap always stays inside: the centre tap
  for (int i = 0; i < d->ntaps; ++i) if (d->taps[i][0] == 0 && d->taps[i][1] == 0 && d->taps[i][2] == 0) p.skip_t = 1;
  p.tiles_x = ceil_div(d->Wo, kTileW); p.tiles_y = ceil_div(d->Ho, kSubH);
  p.stride = d->stride; p.kblocks = kblocks; p.cin_off = d->cin_off; p.ntaps = d->ntaps;
  {
    const int k_lo = d->k_hi > 0 ? d->k_lo : 0, k_hi = d->k_hi > 0 ? d->k_hi : d->cin;
    STP3_CHECK_ARG(k_lo % 16 == 0 && k_hi % 16 == 0 && k_lo >= 0 && k_lo < k_hi && k_hi <= d->cin &&
                   k_lo < kBK && k_hi > d->cin - kBK, "k_lo / k_hi: multiples of 16 inside the first / last 64-channel block");
    p.ks_first = k_lo / 16;
    p.ks_end = (k_hi - (kblocks - 1) * kBK) / 16;
    STP3_CHECK_ARG(kblocks > 1 || p.ks_first < p.ks_end, "empty K range");
  }
  p.a_plane_bytes = t.box_h * kTileW * kBK * 2; p.w_rows = d->bn; p.n_mma = n_mma;
  for (int i = 0; i < d->ntaps; ++i) { p.tap[i][0] = d->taps[i][0]; p.tap[i][1] = d->taps[i][1]; p.tap[i][2] = d->taps[i][2]; p.tap[i][3] = 0; }
  t.k_iters = d->ntaps * kblocks;
  t.full_k = p.ks_first == 0 && p.ks_end == kBK / 16;
  const long long ntile = (long long)p.n_img * p.tiles_x * p.tiles_y;
  STP3_CHECK_ARG(ntile > 0 && ntile * p.n_nblk < (1ll << 31), "grid too large");
  p.n_tiles = (int)ntile;
  const long long items = ntile * p.n_nblk;
  t.grid = (unsigned)(items < n_sm ? items : n_sm);                      // persistent: one CTA per SM

  // ring depths beside this block width's shared-memory tail
  const size_t tail = t.bn_blk == 64 ? ConvSmem<64>::tail_bytes() : ConvSmem<128>::tail_bytes();
  const int planes = operand == 0 ? 2 : 1;
  const size_t a_stage = planes * (size_t)p.a_plane_bytes;
  p.b_rows = t.full_k ? t.bn_blk : n_mma;
  p.b_tile_bytes = planes * p.b_rows * kBK * 2;
  p.b_load_bytes = planes * n_mma * kBK * 2;
  const size_t avail = kSmemCap - 1024 - tail;
  const size_t wbytes = (size_t)t.k_iters * (size_t)p.b_tile_bytes;
  // small weight tensors stay resident in smem next to >= 2 activation stages
  const bool res = !stream_weights && wbytes + 2 * a_stage <= avail;
  int na, nb;
  if (res) {
    na = (int)((avail - wbytes) / a_stage); nb = 0;
  } else {
    // as many activation stages as fit beside two weight slots, then fill up with weight slots (a slot is released
    // one wgmma group after its last reader, so two slots keep a tap group of any size moving)
    na = (int)((avail - 2 * (size_t)p.b_tile_bytes) / a_stage);
    if (na > kMaxAStages) na = kMaxAStages;
    if (na < 2 || (size_t)na * a_stage + 2 * (size_t)p.b_tile_bytes > avail)
      return set_error(STP3_EUNSUPPORTED, "convolution does not fit in shared memory");
    nb = (int)((avail - (size_t)na * a_stage) / (size_t)p.b_tile_bytes);
  }
  if (na > kMaxAStages) na = kMaxAStages;
  if (nb > kMaxBStages) nb = kMaxBStages;
  p.na_stages = na; p.nb_stages = nb; p.b_resident = res ? 1 : 0;
  t.smem_bytes = 1024 + na * a_stage + (res ? wbytes : (size_t)nb * (size_t)p.b_tile_bytes) + tail;
  return STP3_OK;
}

}  // namespace stp3

using namespace stp3;

extern "C" size_t stp3_conv_col_sums_scratch_bytes(int n_img, int bn) {
  return (size_t)num_sms() * 4 * (size_t)(n_img > 0 ? n_img : 0) * (size_t)(bn > 0 ? bn : 0) * sizeof(float);
}

extern "C" int stp3_conv_tiling(const stp3_conv_desc* d, int n_sm, stp3_conv_tiling_info* out) {
  return stp3_conv_tiling_op(d, n_sm, STP3_OPERAND_HILO, out);
}

extern "C" int stp3_conv_tiling_op(const stp3_conv_desc* d, int n_sm, int operand, stp3_conv_tiling_info* out) {
  STP3_CHECK_ARG(d && out && n_sm > 0, "stp3_conv_tiling: null pointer argument or no SM");
  STP3_CHECK_ARG(operand == STP3_OPERAND_HILO || operand == STP3_OPERAND_BF16 || operand == STP3_OPERAND_F16,
                 "stp3_conv_tiling_op: operand must be STP3_OPERAND_HILO, _BF16 or _F16");
  ConvParams p;
  ConvPlan t;
  if (const int rc = plan_conv(d, false, n_sm, p, t, operand)) return rc;
  out->bn_blk = t.bn_blk; out->stacked = t.stack; out->tiles = p.n_tiles; out->items = p.n_tiles * p.n_nblk;
  out->ctas = (int)t.grid; out->a_stages = p.na_stages; out->b_stages = p.nb_stages; out->resident = p.b_resident;
  return STP3_OK;
}

// stp3_conv_fwd and stp3_conv_fwd_plane (operand != 0: x_lo, the residual, the hi/lo outputs and the head are absent)
static int conv_fwd(const stp3_conv_desc* d, int operand, const void* x_hi, const void* x_lo, const void* w,
                    const float* bias, const float* img_bias, const void* res_hi, const void* res_lo, void* y_hi,
                    void* y_lo, float* y_f32, const stp3_conv_head* head, cudaStream_t stream) {
  if (head) {
    STP3_CHECK_ARG(head->n_out >= 1 && head->n_out <= kMaxHeadOut && head->w && head->b, "bad fused head");
    STP3_CHECK_ARG(d->bn <= 128, "a fused head needs bn <= 128");
    for (int k = 0; k < head->n_out; ++k) STP3_CHECK_ARG(head->out[k] != nullptr, "fused head: null output plane");
  }
  ConvParams p;
  ConvPlan t;
  if (const int rc = plan_conv(d, head != nullptr, num_sms(), p, t, operand)) return rc;
  const int n_store = d->n_store > 0 ? d->n_store : d->bn;
  if (y_hi) STP3_CHECK_ARG(d->out_cstride % 8 == 0 && d->out_coff % 8 == 0 && d->out_coff + n_store <= d->out_cstride,
                           "output channel window does not fit the output tensor");
  if (d->res_mode) STP3_CHECK_ARG(res_hi && res_lo && d->res_cstride % 8 == 0 && d->res_coff % 8 == 0 &&
                                  d->res_coff + d->bn <= d->res_cstride, "bad residual tensor");
  if (y_f32) STP3_CHECK_ARG(d->n_valid > 0 && d->n_valid <= d->bn, "n_valid out of range");
  if (!tmap_encode_fn()) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");

  CUtensorMap tm_hi, tm_lo, tm_w;
  {
    const int box_w = (kTileW - 1) * d->stride + 1, box_rows = (t.box_h - 1) * d->stride + 1;
    const CUresult r1 = encode_act_5d(&tm_hi, x_hi, d->in_cstride, d->W, d->H, p.T_total, d->B, box_w, box_rows, d->stride);
    const CUresult r2 = operand ? r1 : encode_act_5d(&tm_lo, x_lo, d->in_cstride, d->W, d->H, p.T_total, d->B, box_w,
                                                     box_rows, d->stride);
    if (operand) tm_lo = tm_hi;
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
      return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation) failed: %d %d", (int)r1, (int)r2);
  }
  {
    const int planes = operand ? 1 : 2;
    const long long rows = d->w_img_stride ? (long long)(d->B * d->T - 1) * (d->w_img_stride / 64) + (long long)t.k_iters * 2 * d->bn
                                           : (long long)t.k_iters * planes * d->bn;
    const CUresult r = encode_rows_2d(&tm_w, w, rows, p.n_mma);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  }

  p.bias = bias; p.img_bias = img_bias; p.img_bias_stride = d->bn;
  p.relu = d->relu; p.res_mode = d->res_mode;
  p.swish = d->swish; p.w_img_rows = d->w_img_stride / 64;
  p.res_hi = static_cast<const __nv_bfloat16*>(res_hi); p.res_lo = static_cast<const __nv_bfloat16*>(res_lo);
  p.res_cstride = d->res_cstride; p.res_coff = d->res_coff;
  p.out_hl = y_hi != nullptr; p.n_store = n_store;
  p.out2 = d->y2_hi != nullptr; p.relu2 = d->relu2;
  const int n_store2 = d->n_store2 > 0 ? d->n_store2 : 64;
  if (d->y2_hi) {
    STP3_CHECK_ARG(d->bn == 128 && d->y2_lo && y_hi && !d->res_mode && !head && !y_f32 && !d->col_sums,
                   "second destination: 128-column convolutions with plain hi/lo outputs only");
    STP3_CHECK_ARG(n_store <= 64 && n_store2 % 8 == 0 && n_store2 <= 64 && d->out2_cstride % 8 == 0 &&
                   d->out2_coff % 8 == 0 && d->out2_coff + n_store2 <= d->out2_cstride,
                   "second destination: channel window does not fit");
  }
  // output maps: primary hi, lo, second destination hi, lo.  Each starts at its destination's channel offset and
  // spans its stored channels, so a tile's TMA store writes nothing outside that window
  CUtensorMap tm_o[4] = {};
  {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    auto enc = [&](CUtensorMap* m, void* plane, int cstride, int coff, int n_ch) {
      return encode_out_4d(m, static_cast<__nv_bfloat16*>(plane) + coff, cstride, n_ch, d->Wo, d->Ho, p.n_img, kTileW, kSubH);
    };
    if (y_hi) {
      STP3_CHECK_ARG(al16(y_hi) && al16(y_lo), "hi/lo output planes must be 16-byte aligned");
      const CUresult r1 = enc(&tm_o[0], y_hi, d->out_cstride, d->out_coff, n_store);
      const CUresult r2 = enc(&tm_o[1], y_lo, d->out_cstride, d->out_coff, n_store);
      if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
        return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(output) failed: %d %d", (int)r1, (int)r2);
    }
    if (d->y2_hi) {
      STP3_CHECK_ARG(al16(d->y2_hi) && al16(d->y2_lo), "second destination planes must be 16-byte aligned");
      const CUresult r1 = enc(&tm_o[2], d->y2_hi, d->out2_cstride, d->out2_coff, n_store2);
      const CUresult r2 = enc(&tm_o[3], d->y2_lo, d->out2_cstride, d->out2_coff, n_store2);
      if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
        return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(second output) failed: %d %d", (int)r1, (int)r2);
    }
  }
  p.out_f32 = y_f32; p.n_valid = d->n_valid; p.sigmoid = d->sigmoid;
  p.f32_nhwc = d->f32_layout;
  if (y_f32 && d->f32_layout == 1)
    STP3_CHECK_ARG((reinterpret_cast<uintptr_t>(y_f32) & 31) == 0 && !d->sigmoid,
                   "channels-last y_f32 must be 32-byte aligned (and carries no sigmoid)");
  p.head_ko = 0; p.head_w = nullptr; p.head_b = nullptr; p.head_sigmoid_mask = 0;
  for (int k = 0; k < kMaxHeadOut; ++k) { p.head_out[k] = nullptr; p.head_img_stride[k] = 0; }
  if (head) {
    p.head_ko = head->n_out; p.head_w = head->w; p.head_b = head->b; p.head_sigmoid_mask = head->sigmoid_mask;
    for (int k = 0; k < head->n_out; ++k) { p.head_out[k] = head->out[k]; p.head_img_stride[k] = head->img_stride[k]; }
  }
  p.sum_part = nullptr;
  if (d->col_sums) {
    STP3_CHECK_ARG(d->bn == 64, "col_sums: 64-column convolutions only");
    STP3_CHECK_ARG(d->col_sums_scratch && d->col_sums_scratch_bytes >= stp3_conv_col_sums_scratch_bytes(p.n_img, 64),
                   "col_sums: scratch buffer missing or smaller than stp3_conv_col_sums_scratch_bytes()");
    p.sum_part = static_cast<float*>(d->col_sums_scratch);
    // CTAs that never see an image leave its partial rows untouched: start from zeros
    STP3_CUDA_OK(cudaMemsetAsync(p.sum_part, 0, (size_t)t.grid * 4 * p.n_img * 64 * sizeof(float), stream));
  }
  // every column block starts a multiple of 64 channels further: one alignment answer for all of them
  auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
  p.vec256 = d->res_mode && d->res_cstride % 16 == 0 && d->res_coff % 16 == 0 && al32(res_hi) && al32(res_lo) ? 2 : 0;
  int rc;
  if (operand == STP3_OPERAND_BF16 && t.bn_blk == 64)
    rc = t.full_k ? launch_conv<64, false, true, 1>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<64, false, false, 1>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else if (operand == STP3_OPERAND_BF16)
    rc = t.full_k ? launch_conv<128, false, true, 1>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<128, false, false, 1>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else if (operand == STP3_OPERAND_F16 && t.bn_blk == 64)
    rc = t.full_k ? launch_conv<64, false, true, 2>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<64, false, false, 2>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else if (operand == STP3_OPERAND_F16)
    rc = t.full_k ? launch_conv<128, false, true, 2>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<128, false, false, 2>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else if (t.bn_blk == 64 && t.stack)
    rc = t.full_k ? launch_conv<64, true, true>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<64, true, false>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else if (t.bn_blk == 64)
    rc = t.full_k ? launch_conv<64, false, true>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<64, false, false>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  else
    rc = t.full_k ? launch_conv<128, false, true>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream)
                  : launch_conv<128, false, false>(p, tm_hi, tm_lo, tm_w, tm_o, t.smem_bytes, t.grid, stream);
  if (rc) return rc;
  STP3_CUDA_OK(cudaGetLastError());
  if (p.sum_part) {
    STP3_CUDA_OK(launch_pdl(kPdlAux, col_sum_reduce_kernel, dim3(p.n_img), dim3(64, 16), 0, stream,
                            (const float*)p.sum_part, (int)t.grid * 4, p.n_img, 64, static_cast<float*>(d->col_sums)));
  }
  return STP3_OK;
}

extern "C" int stp3_conv_fwd(const stp3_conv_desc* d, const void* x_hi, const void* x_lo, const void* w,
                             const float* bias, const float* img_bias, const void* res_hi, const void* res_lo,
                             void* y_hi, void* y_lo, float* y_f32, const stp3_conv_head* head, void* stream) {
  STP3_CHECK_ARG(d && x_hi && x_lo && w && bias, "stp3_conv_fwd: null pointer argument");
  STP3_CHECK_ARG((y_hi && y_lo) || y_f32 || head, "stp3_conv_fwd: no output tensor");
  return conv_fwd(d, STP3_OPERAND_HILO, x_hi, x_lo, w, bias, img_bias, res_hi, res_lo, y_hi, y_lo, y_f32, head,
                  reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int stp3_conv_fwd_plane(const stp3_conv_desc* d, int operand, const void* x, const void* w,
                                   const float* bias, const float* img_bias, float* y_f32, void* stream) {
  STP3_CHECK_ARG(d && x && w && bias && y_f32, "stp3_conv_fwd_plane: null pointer argument");
  STP3_CHECK_ARG(operand == STP3_OPERAND_BF16 || operand == STP3_OPERAND_F16,
                 "stp3_conv_fwd_plane: operand must be STP3_OPERAND_BF16 or STP3_OPERAND_F16");
  STP3_CHECK_ARG(!d->res_mode && !d->y2_hi && !d->col_sums && !d->swish && !d->w_img_stride,
                 "stp3_conv_fwd_plane: no residual, second destination, col_sums, swish or per-image weights");
  return conv_fwd(d, operand, x, nullptr, w, bias, img_bias, nullptr, nullptr, nullptr, nullptr, y_f32, nullptr,
                  reinterpret_cast<cudaStream_t>(stream));
}
