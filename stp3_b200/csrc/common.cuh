// Shared helpers for libstp3_b200.so (sm_90a only).
#pragma once
#include <cuda.h>
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

// The checks the lift-splat forward and backward share (lift_splat.cu): the descriptor with feat and depth_logits, at
// most max_frames frames per sample.  Fills the BEV quantisation constants (lift_geom.cuh) and returns STP3_OK, or an
// STP3_E* code with the message set; `fn` names the entry point in the null-pointer message.
struct BevQuant;
int check_lift_splat_desc(const char* fn, const stp3_lift_splat_desc* d, const float* feat, const float* depth_logits,
                          int max_frames, BevQuant& q);

// ---------------------------------------------------------------- launch plumbing (launch.cu)
using TmapEncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// cuTensorMapEncodeTiled, fetched from the driver once; null if the driver does not provide it
TmapEncodeFn tmap_encode_fn();
// A channels-last bf16 plane (B, T, H, W, cstride) as a 5-D map with the 128-byte swizzle the wgmma operands use: box
// of 64 channels x box_w x box_h pixels, every `estride`-th column and row
CUresult encode_act_5d(CUtensorMap* m, const void* plane, int cstride, int W, int H, int T, int B, int box_w, int box_h,
                       int estride);
// The channel window [0, n_ch) of a channels-last bf16 output plane (n_img, Ho, Wo, cstride) that starts at `plane`, as
// a 4-D map with the same swizzle: box of 64 channels x box_w x box_h pixels.  A store through it writes neither the
// channels beyond n_ch nor the pixels outside the map
CUresult encode_out_4d(CUtensorMap* m, void* plane, int cstride, int n_ch, int Wo, int Ho, int n_img, int box_w, int box_h);
// Packed weights, `rows` rows of 64 bf16, as a 2-D map with the same swizzle: box of box_rows rows
CUresult encode_rows_2d(CUtensorMap* m, const void* w, long long rows, int box_rows);
// multiprocessor count of the current device (cached per device and host thread)
int num_sms();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per kernel, device and host thread: the call costs
// microseconds on every eager launch.  Keyed on the kernel itself, not its type: instantiations share a signature.
template <auto Kern>
cudaError_t set_max_dynamic_smem(int bytes) {
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev == dev_done) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) dev_done = dev;
  return e;
}

// Debug switches, read once per process: STP3_PDL=0 turns programmatic dependent launch off everywhere,
// STP3_CONV_PDL / STP3_FUSED_PDL / STP3_AUX_PDL = 0 for one kernel family.
enum PdlFamily { kPdlConv = 0, kPdlFused = 1, kPdlAux = 2 };
bool pdl_enabled(PdlFamily family);

// Launch with programmatic stream serialization: the kernel may be scheduled while its predecessor drains; it MUST
// execute griddepcontrol.wait (ptx::griddep_wait) before touching global memory the predecessor produced.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(PdlFamily family, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                       cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled(family) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace stp3

