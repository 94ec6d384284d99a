// Shared helpers for libstp3_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/stp3_b200.h"

namespace stp3 {

// thread-local error text behind stp3_last_error()
char* error_buffer();
int set_error(int code, const char* fmt, ...);

#define STP3_CHECK_ARG(cond, ...)                                  \
  do {                                                             \
    if (!(cond)) return ::stp3::set_error(STP3_EINVAL, __VA_ARGS__); \
  } while (0)

#define STP3_CUDA_OK(expr)                                                                        \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return ::stp3::set_error(STP3_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                               __FILE__, __LINE__);                                               \
  } while (0)

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// col_sums[img][c] = fixed-order sum of the (n_part, n_img, 64) partial rows an epilogue wrote (conv_igemm.cu)
int launch_col_sum_reduce(const float* part, int n_part, int n_img, float* out, cudaStream_t stream);

}  // namespace stp3

// Debug switches: STP3_PDL=0 turns programmatic dependent launch off everywhere, `family`=0 (STP3_CONV_PDL,
// STP3_FUSED_PDL, STP3_AUX_PDL) for one kernel family.
static inline bool stp3_pdl_enabled(const char* family) {
  const char* all = getenv("STP3_PDL");
  if (all && atoi(all) == 0) return false;
  const char* e = getenv(family);
  return !e || atoi(e) != 0;
}

// Launch with programmatic stream serialization: the kernel may be scheduled while its predecessor drains; it MUST
// execute griddepcontrol.wait (ptx::griddep_wait) before touching global memory the predecessor produced.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = stp3_pdl_enabled("STP3_AUX_PDL") ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

