// ASPP branches + 1x1 projection as ONE back-to-back wgmma kernel (DeepLabHead of the temporal model,
// stp3/layers/convolutions.py:242-270: four conv/BN/ReLU branches of the same input, concatenated, then project.0).
//
// The unfused form writes the 4 x 128-channel concat tensor to HBM (4 x 246 MB for a 4-sample step) and reads it back
// (984 MB) -- the largest avoidable traffic of the dense path.  Here a CTA keeps an 8x16-pixel tile on chip:
//
//   for every branch b:   acc1  = sum_taps A(x, tap) . W_b[tap]            (wgmma, 64 rows per warpgroup, N = 128)
//                         P     = hi/lo split of relu(acc1 + bias_b)       (in registers: the accumulator fragment,
//                                                                           packed to bf16x2, is the wgmma A fragment)
//                         acc2 += P . W_proj[:, b-th 128 input channels]   (second MMA chain, A operand = P from registers)
//   out = hi/lo split of relu(acc2 + per-image bias)                       (the global-pool branch is that bias)
//
// The output tile is staged in the activation stage the last branch's last tap read, laid out as the TMA load wrote it
// (per plane [pixel row][128 B], 128-byte swizzle), one 64-channel block at a time, and leaves by one
// cp.async.bulk.tensor store per warpgroup, plane and block.  That stage goes back to the producer once the stores have
// read it, early in the next tile, whose first taps load into the other two stages.
//
// The same kernel runs the head's tail, 3x3 conv/BN/ReLU -> 1x1 classifier (convolutions.py:272-280), as a ONE-branch
// instance (9 taps, two input K blocks, classifier rows padded to 128, no ReLU on the output).
//
// Same precision scheme as conv_igemm.cu (bf16 hi/lo planes, hi*hi + hi*lo + lo*hi, fp32 accumulation), so the result
// matches the unfused path to the last few bits of the split.
//
//   warps : 0..7 = two warpgroups (rows 0..63 / 64..127 of the tile), 8 = TMA producer (activation ring + weight ring),
//           9..11 idle.  The producer warpgroup hands its registers to the MMA warpgroups (setmaxnreg 40 / 232): acc1,
//           acc2 and P live at once do not fit the 168 registers per thread of an even split
//   smem  : 3 activation stages (96 KB) + 3 weight stages (96 KB) = 192 KB.  P never touches shared memory, so both rings
//           are three deep: a step's operands are requested two MMA steps before they are used (with two stages, one
//           step of MMAs had to cover the whole TMA latency)
#include <cuda_bf16.h>

#include "common.cuh"
#include "pipeline.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace stp3 {

constexpr int kAsppThreads = 384;                 // 8 + 4 warps
constexpr int kAsppMaxBranches = 4;
constexpr int kAsppMaxTaps = 9 * kAsppMaxBranches;
constexpr int kAsppNA = 3, kAsppNB = 3;
constexpr int kAStage = 2 * 8 * 16 * 128;         // hi + lo planes of 8 image rows x 16 pixels x 64 channels
constexpr int kBStage = 2 * 128 * 128;            // hi + lo planes of the 128 weight rows
constexpr int kAsppHidden = 128;
// the output tile is staged in an activation stage: per plane 128 pixel rows of 128 bytes (64 channels), 1024-byte
// aligned for the 128-byte swizzle; each warpgroup stores its 64 rows as one box of 16 x kAsppStoreRows pixels
constexpr int kAsppStoreRows = 4;
static_assert(kAStage / 2 == 8 * 16 * 128 && (kAStage / 2) % 1024 == 0, "an activation plane stages 128 pixels x 64 channels");
static_assert(16 * kAsppStoreRows == 64, "one store box per warpgroup: its 64 accumulator rows");

// shared memory, from the 1024-byte aligned base (the kernel carves it, the host sizes the launch from `bytes`)
struct AsppSmem {
  static constexpr int a_ring = 0;                                          // kAsppNA activation stages
  static constexpr int b_ring = a_ring + kAsppNA * kAStage;                 // kAsppNB weight stages
  static constexpr int bias = b_ring + kAsppNB * kBStage;                   // fp32 [kAsppMaxBranches][128] branch biases
  static constexpr int wb = bias + kAsppMaxBranches * kAsppHidden * 4;      // fp32 [2 warpgroups][128] per-image bias
  static constexpr int bars = wb + 2 * kAsppHidden * 4;                     // full / empty barriers of both rings
  static constexpr size_t bytes = 1024 + bars + 2 * (kAsppNA + kAsppNB) * 8;   // + the alignment slack
};

struct AsppParams {
  int n_img, T, T_total, H, W;
  int tiles_x, tiles_y, n_tiles;
  int kblocks;
  int n_br;
  int br_tap0[kAsppMaxBranches + 1];
  signed char tap[kAsppMaxTaps][2];               // (dy, dx)
  const float* br_bias;                           // [n_br][128]
  const float* img_bias;                          // [n_img][128]
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
                  const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_o_hi,
                  const __grid_constant__ CUtensorMap tm_o_lo, const AsppParams p) {
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* a_ring = smem + AsppSmem::a_ring;
  unsigned char* b_ring = smem + AsppSmem::b_ring;
  float* s_bias = reinterpret_cast<float*>(smem + AsppSmem::bias);
  float* s_wb = reinterpret_cast<float*>(smem + AsppSmem::wb);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AsppSmem::bars);
  Ring ra{bars, bars + kAsppNA, kAsppNA};
  Ring rb{bars + 2 * kAsppNA, bars + 2 * kAsppNA + kAsppNB, kAsppNB};

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    ptx::prefetch_tmap(&tm_a_hi); ptx::prefetch_tmap(&tm_a_lo); ptx::prefetch_tmap(&tm_w);
    ptx::prefetch_tmap(&tm_o_hi); ptx::prefetch_tmap(&tm_o_lo);
    ra.init(2); rb.init(2);
    ptx::fence_mbar_init();
  }
  for (int i = threadIdx.x; i < p.n_br * kAsppHidden; i += blockDim.x) s_bias[i] = p.br_bias[i];
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int proj_blk0 = p.br_tap0[p.n_br] * p.kblocks;          // first projection block of the weight tensor

  if (warp >= 8) {
    ptx::setmaxnreg_dec<40>();
    if (warp != 8) return;
    // ===================== TMA producer =====================
    ptx::griddep_wait();
    auto load_b = [&](int blk) {                   // weight block `blk`: [hi 128 rows][lo 128 rows]
      rb.produce(kBStage, [&](int s, uint64_t* bar) {
        unsigned char* dst = b_ring + (size_t)s * kBStage;
        ptx::tma_load_2d(dst, &tm_w, bar, 0, blk * 256);
        ptx::tma_load_2d(dst + 128 * 128, &tm_w, bar, 0, blk * 256 + 128);
      });
    };
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      const int bidx = img / p.T, tidx = img % p.T;
      for (int s = 0; s < p.n_br; ++s) {
        for (int t = p.br_tap0[s]; t < p.br_tap0[s + 1]; ++t) {
          if (aspp_tap_is_padding(p, t, oy_tile, ox0)) continue;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            ra.produce(kAStage, [&](int s, uint64_t* bar) {
              unsigned char* sa = a_ring + (size_t)s * kAStage;
              ptx::tma_load_5d(sa, &tm_a_hi, bar, kb * 64, ox0 + p.tap[t][1], oy_tile + p.tap[t][0], tidx, bidx);
              ptx::tma_load_5d(sa + kAStage / 2, &tm_a_lo, bar, kb * 64, ox0 + p.tap[t][1], oy_tile + p.tap[t][0], tidx, bidx);
            });
            load_b(t * p.kblocks + kb);
          }
        }
        load_b(proj_blk0 + s * 2); load_b(proj_blk0 + s * 2 + 1);   // projection weights of this branch
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // ===================== two warpgroups: branch MMAs, conversion to P, projection, output =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int wtid = threadIdx.x & 127;
    const int row0 = wg * 64 + wq * 16 + (lane >> 2);       // accumulator rows of this thread: row0, row0 + 8
    const int cq = 2 * (lane & 3);                           // first of its two columns in every 8-column group
    float* wb = s_wb + wg * kAsppHidden;
    PendingSlots pend{ra.empty, rb.empty, wtid == 0};
    int out_slot = -1;                           // activation stage holding the previous tile's output until stored
    // acc (+)= A . B over one 64-channel K block, then commit, release the previous group's slots, and the previous
    // tile's output stage once its stores have read it (the new group runs meanwhile)
    auto issue = [&](float* acc, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, uint32_t accumulate,
                     int slot_a, int slot_b) {
      const uint64_t da_hi = wg::desc_k_sw128(a_hi), da_lo = wg::desc_k_sw128(a_lo);
      const uint64_t db_hi = wg::desc_k_sw128(b_hi), db_lo = wg::desc_k_sw128(b_lo);
      wg::fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t koff = (uint64_t)((k * 32) >> 4);
        wg::mma_hilo<kAsppHidden>(acc, da_hi + koff, da_lo + koff, db_hi + koff, db_lo + koff, accumulate | (uint32_t)k);
      }
      wg::commit();
      wg::wait<1>();
      pend.release_and_defer(slot_a, slot_b);
      if (out_slot >= 0) {
        if (wtid == 0) { ptx::bulk_wait_read0(); ptx::mbar_arrive(&ra.empty[out_slot]); }
        out_slot = -1;
      }
    };
    ptx::griddep_wait();
    for (int tile = cta; tile < p.n_tiles; tile += n_cta) {
      const int img = tile / tiles_per_img, rem = tile % tiles_per_img;
      const int oy_tile = (rem / p.tiles_x) * 8, ox0 = (rem % p.tiles_x) * 16;
      ptx::bar_sync(1 + wg, 128);                // the previous tile's output has read the per-image bias
      // written by the preceding (PDL-overlapped) pool_bias kernel: coherent loads
      wb[wtid] = *(reinterpret_cast<const volatile float*>(p.img_bias) + (size_t)img * kAsppHidden + wtid);
      ptx::bar_sync(1 + wg, 128);                // the output reads entries other warps of the warpgroup wrote
      float acc2[kAsppHidden / 2];
      int stage = -1;                            // the last branch's last activation stage: the output staging area
      for (int s = 0; s < p.n_br; ++s) {
        // ---- main(s): acc1 = sum over the branch's taps
        float acc1[kAsppHidden / 2];
        uint32_t accumulate = 0;
        for (int t = p.br_tap0[s]; t < p.br_tap0[s + 1]; ++t) {
          if (aspp_tap_is_padding(p, t, oy_tile, ox0)) continue;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            ra.wait_full();
            rb.wait_full();
            const uint32_t a_hi = ptx::smem_u32(a_ring + (size_t)ra.slot * kAStage) + (uint32_t)(wg * 64 * 128);
            const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)rb.slot * kBStage);
            issue(acc1, a_hi, a_hi + kAStage / 2, b_hi, b_hi + 128 * 128, accumulate, ra.slot, rb.slot);
            accumulate = 1;
            ra.advance();
            rb.advance();
          }
        }
        wg::wait<0>();                             // also: the previous branch's projection has read P's registers
        if (s + 1 == p.n_br) { stage = pend.a; pend.a = -1; }   // the centre tap is never padding: a stage was read
        pend.release();
        // ---- P = hi/lo split of relu(acc1 + bias), kept in registers, and proj(s): acc2 (+)= P . W_proj[:, branch s],
        // one 64-column K block kb2 at a time.  Accumulator entries (4 g8 + 2 h, +1) -- row row0 + 8 h, columns
        // 8 g8 + cq, +1 -- become bf16x2 register 2 (g8 % 8) + h, and registers 4 k .. 4 k + 3 are the A fragment of the
        // block's columns 16 k .. 16 k + 15 (wgmma.cuh, mma_bf16_rs128).  Converting per block lets each half of acc1
        // die as its half of P is made: acc1, acc2 and all of P would exceed the 168 registers a thread of this
        // 288-thread kernel gets, and ptxas would serialise every wgmma.
        const float* bias = s_bias + s * kAsppHidden;
#pragma unroll
        for (int kb2 = 0; kb2 < 2; ++kb2) {
          uint32_t p_hi[16], p_lo[16];
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const int g8 = 8 * kb2 + g;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float x0 = fmaxf(acc1[4 * g8 + 2 * h] + bias[8 * g8 + cq], 0.f);
              const float x1 = fmaxf(acc1[4 * g8 + 2 * h + 1] + bias[8 * g8 + cq + 1], 0.f);
              ptx::split_hilo(x0, x1, p_hi[2 * g + h], p_lo[2 * g + h]);
            }
          }
          rb.wait_full();
          const uint32_t b_hi = ptx::smem_u32(b_ring + (size_t)rb.slot * kBStage);
          const uint64_t db_hi = wg::desc_k_sw128(b_hi), db_lo = wg::desc_k_sw128(b_hi + 128 * 128);
          wg::fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t koff = (uint64_t)((k * 32) >> 4);
            wg::mma_hilo_rs<kAsppHidden>(acc2, &p_hi[4 * k], &p_lo[4 * k], db_hi + koff, db_lo + koff,
                                         (s > 0 || kb2 > 0 || k > 0) ? 1u : 0u);
          }
          wg::commit();
          wg::wait<0>();                           // P's registers are read until the group completes
          pend.release_and_defer(-1, rb.slot);
          rb.advance();
        }
      }
      wg::wait<0>();
      pend.release();
      // ---- output of the projection: relu(acc2 + per-image bias) -> hi/lo planes, one 64-channel block at a time
      // through the staging stage: row r of this warpgroup's 64 at r * 128 bytes of each plane, 16-byte chunk g at
      // chunk g ^ (r & 7).  The second block waits until the first block's stores have read the stage
      unsigned char* st_hi = a_ring + (size_t)stage * kAStage;
      unsigned char* st_lo = st_hi + kAStage / 2;
      const uint32_t src = ptx::smem_u32(st_hi) + (uint32_t)(wg * 64 * 128);
#pragma unroll
      for (int cb = 0; cb < kAsppHidden / 64; ++cb) {
        if (cb * 64 >= p.n_store) break;
        if (cb > 0) {
          if (wtid == 0) ptx::bulk_wait_read0();
          ptx::bar_sync(1 + wg, 128);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const int g8 = 8 * cb + g, c = 8 * g8 + cq;
            float x0 = acc2[4 * g8 + 2 * h] + wb[c];
            float x1 = acc2[4 * g8 + 2 * h + 1] + wb[c + 1];
            if (p.relu_out) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            uint32_t hw, lw;
            ptx::split_hilo(x0, x1, hw, lw);
            const uint32_t off = (uint32_t)(row * 128 + ((g ^ (row & 7)) << 4) + 2 * cq);
            *reinterpret_cast<uint32_t*>(st_hi + off) = hw;
            *reinterpret_cast<uint32_t*>(st_lo + off) = lw;
          }
        }
        ptx::fence_proxy_async();                // the generic-proxy writes are visible to the TMA stores
        ptx::bar_sync(1 + wg, 128);              // every row of this warpgroup's half is written
        if (wtid == 0) {                         // image rows oy_tile + 4 wg .. + 3: the map clips the ragged edges
          ptx::tma_store_4d(&tm_o_hi, src, cb * 64, ox0, oy_tile + kAsppStoreRows * wg, img);
          ptx::tma_store_4d(&tm_o_lo, src + kAStage / 2, cb * 64, ox0, oy_tile + kAsppStoreRows * wg, img);
          ptx::bulk_commit();
        }
      }
      out_slot = stage;
    }
    if (wtid == 0) ptx::bulk_wait0();            // the last tile's outputs are written before the CTA exits
  }
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
  p.relu_out = d->no_relu ? 0 : 1; p.n_store = n_store;
  // every descriptor check comes before the driver lookup: a bad descriptor is reported as such without a GPU
  if (!tmap_encode_fn()) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");

  CUtensorMap tm_hi, tm_lo, tm_w, tm_o[2];
  {
    const CUresult r1 = encode_act_5d(&tm_hi, x_hi, d->in_cstride, d->W, d->H, d->T, d->B, 16, 8, 1);
    const CUresult r2 = encode_act_5d(&tm_lo, x_lo, d->in_cstride, d->W, d->H, d->T, d->B, 16, 8, 1);
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS)
      return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(activation) failed: %d %d", (int)r1, (int)r2);
    const CUresult r3 = encode_rows_2d(&tm_w, w, (long long)(t * p.kblocks + 2 * d->n_br) * 256, 128);
    if (r3 != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r3);
  }
  void* outs[2] = {y_hi, y_lo};
  for (int i = 0; i < 2; ++i) {       // the n_store-channel output window; one box = one warpgroup's 4 x 16 pixels
    const CUresult r = encode_out_4d(&tm_o[i], static_cast<__nv_bfloat16*>(outs[i]) + d->out_coff, d->out_cstride, n_store,
                                     d->W, d->H, p.n_img, 16, kAsppStoreRows);
    if (r != CUDA_SUCCESS) return set_error(STP3_ECUDA, "cuTensorMapEncodeTiled(output %d) failed: %d", i, (int)r);
  }
  STP3_CUDA_OK(set_max_dynamic_smem<aspp_fused_kernel>((int)AsppSmem::bytes));
  const int n_sm = num_sms();
  // The kernel never executes griddepcontrol.launch_dependents: its dependents are released when the grid completes
  // (see block_fused.cu); it still starts early behind its predecessor.
  STP3_CUDA_OK(launch_pdl(kPdlFused, aspp_fused_kernel, dim3((unsigned)(nt < n_sm ? nt : n_sm)), dim3(kAsppThreads),
                          AsppSmem::bytes, stream, tm_hi, tm_lo, tm_w, tm_o[0], tm_o[1], p));
  STP3_CUDA_OK(cudaGetLastError());
  return STP3_OK;
}
