// univl_b200 — host-side TMA tensor-map construction shared by the wgmma kernels' launchers.
#pragma once

#include "common.cuh"

namespace univl {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  // libcuda is resolved at run time through the runtime (the .so does not link it, so it loads on GPU-less hosts)
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2D bf16 (or, with e4m3, 1-byte) tensor map over a row-major [rows, cols] matrix with leading dimension ld
// (elements); box = {128 B of columns (64 bf16 or 128 e4m3, swizzled), box_rows}.
static inline int make_tmap(CUtensorMap* tm, const void* ptr, long long rows, long long cols, long long ld, int box_rows,
                            bool e4m3 = false) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(UNIVL_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  const int esize = e4m3 ? 1 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, e4m3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(UNIVL_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld ptr=%p", (int)r,
                     rows, cols, ld, ptr);
  return UNIVL_OK;
}

// tensor map of an epilogue operand: row-major [rows, cols] of bf16 or fp32, box = 32 rows x 128 bytes, 128B swizzle
static inline int make_tmap_epi(CUtensorMap* tm, const void* ptr, bool f32, long long rows, long long cols, long long ld) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(UNIVL_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  const int esize = f32 ? 4 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), 32};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(UNIVL_ERR_CUDA, "cuTensorMapEncodeTiled(epilogue) failed (%d) rows=%lld cols=%lld ld=%lld ptr=%p",
                     (int)r, rows, cols, ld, ptr);
  return UNIVL_OK;
}

}  // namespace univl
