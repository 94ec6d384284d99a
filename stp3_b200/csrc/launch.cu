// Host-side launch plumbing shared by the TMA kernels: the tensor-map encoder, the SM count and the PDL switches.
#include <cstdlib>

#include "common.cuh"

namespace stp3 {

TmapEncodeFn tmap_encode_fn() {
  static const TmapEncodeFn fn = [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<TmapEncodeFn>(ptr);
    return TmapEncodeFn(nullptr);
  }();
  return fn;
}

CUresult encode_act_5d(CUtensorMap* m, const void* plane, int cstride, int W, int H, int T, int B, int box_w, int box_h,
                       int estride) {
  const TmapEncodeFn enc = tmap_encode_fn();
  if (!enc) return CUDA_ERROR_NOT_FOUND;
  const cuuint64_t dims[5] = {(cuuint64_t)cstride, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)T, (cuuint64_t)B};
  const cuuint64_t strides[4] = {(cuuint64_t)cstride * 2, (cuuint64_t)W * cstride * 2, (cuuint64_t)H * W * cstride * 2,
                                 (cuuint64_t)T * H * W * cstride * 2};
  const cuuint32_t box[5] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
  const cuuint32_t es[5] = {1, (cuuint32_t)estride, (cuuint32_t)estride, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(plane), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

CUresult encode_out_4d(CUtensorMap* m, void* plane, int cstride, int n_ch, int Wo, int Ho, int n_img, int box_w, int box_h) {
  const TmapEncodeFn enc = tmap_encode_fn();
  if (!enc) return CUDA_ERROR_NOT_FOUND;
  const cuuint64_t dims[4] = {(cuuint64_t)n_ch, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)n_img};
  const cuuint64_t strides[3] = {(cuuint64_t)cstride * 2, (cuuint64_t)Wo * cstride * 2, (cuuint64_t)Ho * Wo * cstride * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, plane, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

CUresult encode_rows_2d(CUtensorMap* m, const void* w, long long rows, int box_rows) {
  const TmapEncodeFn enc = tmap_encode_fn();
  if (!enc) return CUDA_ERROR_NOT_FOUND;
  const cuuint64_t dims[2] = {64, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {128};
  const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  const cuuint32_t es[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

int num_sms() {
  static thread_local int dev_cached = -1, n = 132;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != dev_cached) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    dev_cached = dev;
  }
  return n;
}

bool pdl_enabled(PdlFamily family) {
  auto on = [](const char* name) { const char* e = getenv(name); return !e || atoi(e) != 0; };
  static const bool all = on("STP3_PDL");
  static const bool fam[3] = {all && on("STP3_CONV_PDL"), all && on("STP3_FUSED_PDL"), all && on("STP3_AUX_PDL")};
  return fam[family];
}

}  // namespace stp3
