// Host-side TMA descriptor construction.  The driver entry point is resolved at run time through the
// CUDA runtime so the extension never links against libcuda (it must also build on GPU-less hosts).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

namespace tb {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || p == nullptr || q != cudaDriverEntryPointSuccess)
      throw std::runtime_error("torchacc_b200: cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// Rank-N row-major tensor map; dims/strides are given innermost-first (dims[0] is contiguous).
// strides_bytes has rank-1 entries (stride of dims[1..]).
inline CUtensorMap make_tensor_map(const void* base, CUtensorMapDataType dtype, int rank, const uint64_t* dims,
                                   const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle,
                                   CUtensorMapL2promotion l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_256B) {
  CUtensorMap m;
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  CUresult r = get_encode_tiled()(&m, dtype, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) {
    // Driver entry points need a current context on THIS thread; autograd's backward threads may not have touched
    // the runtime yet.  cudaFree(0) binds the device's primary context, then retry.
    cudaFree(0);
    r = get_encode_tiled()(&m, dtype, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS)
    throw std::runtime_error("torchacc_b200: cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return m;
}

// 2-D bf16 matrix [rows][cols] (cols contiguous, row pitch ld elements), SWIZZLE_128B boxes.
inline CUtensorMap make_map_2d_bf16(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols,
                                    uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * 2};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tensor_map(base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// 2-D fp32 matrix [rows][cols] (cols contiguous, row pitch ld elements), SWIZZLE_128B boxes (box_cols <= 32).
inline CUtensorMap make_map_2d_f32(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols,
                                   uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * 4};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tensor_map(base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace tb
