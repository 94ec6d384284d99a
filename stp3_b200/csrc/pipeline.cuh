// The TMA operand ring of the wgmma kernels (conv_igemm.cu, aspp_fused.cu, block_fused.cu): `stages` shared-memory
// slots, each with a full barrier (one arrive.expect_tx by the producer + the TMA transaction bytes) and an empty
// barrier (one arrive per consumer warpgroup once its wgmma have read the slot).  The producer warp and every consumer
// thread keep their own copy of the ring and walk the slots in the same order.
#pragma once
#include <cstdint>

#include "ptx.cuh"

namespace stp3 {

struct Ring {
  uint64_t* full;
  uint64_t* empty;
  int stages;
  int slot = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ void init(uint32_t consumers) const {     // one thread, before fence_mbar_init
    for (int i = 0; i < stages; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], consumers); }
  }
  __device__ __forceinline__ void advance() {
    if (++slot == stages) { slot = 0; phase ^= 1; }
  }
  // producer step (whole warp): wait until the slot is free, one elected lane posts `bytes` and issues the loads
  // load(slot, full barrier), then advance
  template <class Load>
  __device__ __forceinline__ void produce(uint32_t bytes, Load&& load) {
    ptx::mbar_wait(&empty[slot], phase ^ 1);
    if (ptx::elect_one_sync()) {
      ptx::mbar_arrive_expect_tx(&full[slot], bytes);
      load(slot, &full[slot]);
    }
    __syncwarp();
    advance();
  }
  __device__ __forceinline__ void wait_full() const { ptx::mbar_wait(&full[slot], phase); }
};

// Consumer side: the A and B slots the last committed wgmma group reads (-1: none, or not released by this group).  They
// are released once the next group has been committed and wgmma.wait_group has retired the reading one, so the tensor
// pipe always has the next group queued; the warpgroup leader arrives for its warpgroup.
struct PendingSlots {
  uint64_t* a_empty;
  uint64_t* b_empty;
  bool leader;
  int a = -1, b = -1;

  __device__ __forceinline__ void release() {
    if (leader) {
      if (a >= 0) ptx::mbar_arrive(&a_empty[a]);
      if (b >= 0) ptx::mbar_arrive(&b_empty[b]);
    }
    a = b = -1;
  }
  // after wgmma.wait_group 1 of a newly committed group that reads slots (slot_a, slot_b)
  __device__ __forceinline__ void release_and_defer(int slot_a, int slot_b) {
    release();
    a = slot_a; b = slot_b;
  }
};

}  // namespace stp3
