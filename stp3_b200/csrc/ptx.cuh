// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), programmatic dependent launch, setmaxnreg.
#pragma once
#include <cstdint>
#include <cuda.h>  // CUtensorMap (types only; the encode entry point is fetched at run time)
#include <cuda_bf16.h>

namespace stp3 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// two fp32 -> packed bf16x2 (round to nearest even): low half = a, high half = b
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// two fp32 -> packed f16x2 (round to nearest even; overflow gives +-inf, NaN stays NaN): low half = a, high half = b
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// the one-plane formats of the autocast train path (OP 1 = bf16, 2 = fp16), rounded to nearest even, never saturated
template <int OP>
__device__ __forceinline__ uint32_t pack_plane16x2(float a, float b) {
  static_assert(OP == 1 || OP == 2, "one-plane kind: 1 = bf16, 2 = fp16");
  if constexpr (OP == 2) return pack_f16x2(a, b);
  else return pack_bf16x2(a, b);
}
template <int OP>
__device__ __forceinline__ uint16_t plane16(float x) { return (uint16_t)(pack_plane16x2<OP>(x, 0.f) & 0xFFFFu); }

// The hi/lo plane format of every fp32 tensor: hi = bf16(x), lo = bf16(x - hi), both rounded to nearest even.
// A pair (x0, x1) -> packed bf16x2 words, x0 in the low halves.
__device__ __forceinline__ void split_hilo(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(x0, x1);
  lo = pack_bf16x2(x0 - __uint_as_float(hi << 16), x1 - __uint_as_float(hi & 0xFFFF0000u));
}
// one element (the same rounding as the pair form)
__device__ __forceinline__ void split_hilo(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// hi + lo of the low and the high halves of a packed pair
__device__ __forceinline__ float2 join_hilo(uint32_t hi, uint32_t lo) {
  return make_float2(__uint_as_float(hi << 16) + __uint_as_float(lo << 16),
                     __uint_as_float(hi & 0xFFFF0000u) + __uint_as_float(lo & 0xFFFF0000u));
}

// 32-byte global accesses (8 x 32 bit) as two 128-bit instructions: Hopper has no 256-bit load / store.  16-byte aligned.
__device__ __forceinline__ void ld_global_nc_v8(const void* p, uint32_t (&v)[8]) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\tld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
               : "l"(p));
}
__device__ __forceinline__ void ld_global_v8(const void* p, uint32_t (&v)[8]) {      // coherent (data written earlier)
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%8];\n\tld.global.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
               : "l"(p)
               : "memory");
}
__device__ __forceinline__ uint4 ld_global_v4(const void* p) {                        // coherent 128-bit load
  uint4 r;
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_global_v8(void* p, const uint32_t (&v)[8]) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};\n\tst.global.v4.b32 [%0+16], {%5,%6,%7,%8};" ::"l"(p), "r"(v[0]),
               "r"(v[1]), "r"(v[2]), "r"(v[3]), "r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7])
               : "memory");
}

__device__ __forceinline__ void st_global_v8f(void* p, const float* v) {             // 8 consecutive floats, 16-byte aligned
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};\n\tst.global.v4.f32 [%0+16], {%5,%6,%7,%8};" ::"l"(p), "f"(v[0]),
               "f"(v[1]), "f"(v[2]), "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
               : "memory");
}

// true in exactly one (elected) lane of a converged warp (TMA issue goes through the uniform datapath)
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .b32 rx;\n\t"
      ".reg .pred px;\n\t"
      "elect.sync rx|px, 0xFFFFFFFF;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch
// launch_dependents: the next kernel of the stream (launched with programmatic stream serialization) may start its
// prologue once every CTA of this grid has passed this point or exited.  wait: blocks until the preceding grid has
// completed and flushed its memory; everything that reads or writes dependent global memory comes after it.  Both
// are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// shared::cta -> global tensor store of one box (4-D map), tracked by the issuing thread's bulk groups.  Elements of
// the box outside the map's bounds are not written.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk group of this thread has finished reading its shared-memory source (the buffer may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every bulk group of this thread has completed, its global writes included
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// warpgroup register reallocation (every warp of the warpgroup executes it): lower / raise this warpgroup's per-thread
// register count to N
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// named barrier over `count` threads (a multiple of 32) of the CTA
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// arrive without waiting: a producer's half of a named-barrier hand-over whose consumers bar_sync on the same id
__device__ __forceinline__ void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

}  // namespace ptx
}  // namespace stp3
