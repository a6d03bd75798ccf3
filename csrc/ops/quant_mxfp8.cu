// MX-FP8 quantiser: bf16 -> e4m3 elements + one UE8M0 scale per 32 elements, in the layouts gemm_mxfp8.cu consumes.
//
// One pass over x[R][C] can produce BOTH orientations (every operand of a linear layer is needed twice, with the scales
// running along a different dimension each time -- forward / dgrad contract over features, wgrad over tokens):
//   q  [R][C] + sf  : scales along C   (x as a K-major operand whose K is C)
//   qt [C][R] + sft : scales along R   (x^T as a K-major operand whose K is R: "transpose-requantise")
// Scale tensors are written in the tensor core's atom order (cutlass Sm1xxBlockScaledBasicChunk): atom (row block of
// 128, K block of 128 elements) = 512 bytes, byte (r % 32) * 16 + ((r % 128) / 32) * 4 + (kblock % 4); atoms are stored
// [row block][K atom].  Scale = 2^ceil(log2(amax / 448)) (no saturation), element = round-to-nearest-even e4m3.
// Non-finite input: amax skips NaN (fmaxf), so a NaN element becomes NaN alone; an infinite amax clamps the scale byte
// at 254, whose inverse scale is 0, so the block's finite elements become +-0 and the infinity NaN
// (fp8.quantize_mxfp8_ref emulates both).
//
// The reference has no fp8 support (torchacc/config.py:27-54).
#include <cuda_fp8.h>

#include "../common/ptx.cuh"
#include "ops.h"

namespace tb {

namespace {

constexpr int kTile = 128;
constexpr int kPitch = kTile + 8;     // bf16 elements per smem row (+16 bytes: column walks hit different banks)

__device__ __forceinline__ uint32_t e8m0_from_amax(float amax) {
  if (!(amax > 0.f)) return 0u;
  const float x = amax * (1.0f / 448.0f);
  const uint32_t bits = __float_as_uint(x);
  uint32_t e = (bits >> 23) & 0xffu;
  if (bits & 0x7fffffu) e += 1;               // round the exponent up: scale >= amax / 448
  if (e == 0) e = 1;                          // denormal x: smallest normal scale is plenty
  return e > 254u ? 254u : e;
}
__device__ __forceinline__ float inv_scale_from_e8m0(uint32_t e) {   // 2^(127 - e)
  return __uint_as_float((254u - e) << 23);
}
__device__ __forceinline__ uint32_t pack4_e4m3(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}

__global__ void __launch_bounds__(256)
quant_mxfp8_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int R, int C, uint8_t* __restrict__ q,
                   long long ldq, uint8_t* __restrict__ sf, int sf_katoms, uint8_t* __restrict__ qt, long long ldqt,
                   uint8_t* __restrict__ sft, int sft_katoms) {
  __shared__ __align__(16) __nv_bfloat16 tile[kTile * kPitch];
  const int tr = blockIdx.y, tc = blockIdx.x;
  const int r0 = tr * kTile, c0 = tc * kTile;
  // ---- load the 128 x 128 tile (zero beyond the edges) ----
  for (int i = threadIdx.x; i < kTile * (kTile / 8); i += blockDim.x) {
    const int r = i / (kTile / 8), v = i % (kTile / 8);
    uint4 val = make_uint4(0, 0, 0, 0);
    if (r0 + r < R && c0 + v * 8 + 8 <= C)
      val = *reinterpret_cast<const uint4*>(x + (long long)(r0 + r) * ldx + c0 + v * 8);
    else if (r0 + r < R) {
      __nv_bfloat16 tmp[8];
      for (int j = 0; j < 8; ++j)
        tmp[j] = (c0 + v * 8 + j < C) ? x[(long long)(r0 + r) * ldx + c0 + v * 8 + j] : __float2bfloat16(0.f);
      val = *reinterpret_cast<uint4*>(tmp);
    }
    *reinterpret_cast<uint4*>(&tile[r * kPitch + v * 8]) = val;
  }
  __syncthreads();
  // ---- row-wise: (row, block of 32 columns) pairs ----
  if (q != nullptr) {
    for (int p = threadIdx.x; p < kTile * 4; p += blockDim.x) {
      const int r = p >> 2, b = p & 3;
      float v[32];
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] = __bfloat162float(tile[r * kPitch + b * 32 + j]);
        amax = fmaxf(amax, fabsf(v[j]));
      }
      const uint32_t e = e8m0_from_amax(amax);
      const float inv = inv_scale_from_e8m0(e);
      if (r0 + r < R) {
        uint32_t w[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = pack4_e4m3(v[4 * j] * inv, v[4 * j + 1] * inv, v[4 * j + 2] * inv, v[4 * j + 3] * inv);
        uint8_t* dst = q + (long long)(r0 + r) * ldq + c0 + b * 32;
        if (c0 + b * 32 + 32 <= C) {
          reinterpret_cast<uint4*>(dst)[0] = make_uint4(w[0], w[1], w[2], w[3]);
          reinterpret_cast<uint4*>(dst)[1] = make_uint4(w[4], w[5], w[6], w[7]);
        } else {
          for (int j = 0; j < 32; ++j)
            if (c0 + b * 32 + j < C) dst[j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
      }
      sf[((size_t)tr * sf_katoms + tc) * 512 + (r & 31) * 16 + (r >> 5) * 4 + b] = (uint8_t)e;
    }
  }
  // ---- column-wise (transposed output): (column, block of 32 rows) pairs ----
  if (qt != nullptr) {
    for (int p = threadIdx.x; p < kTile * 4; p += blockDim.x) {
      const int c = p & (kTile - 1), b = p >> 7;          // consecutive threads -> consecutive columns
      float v[32];
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] = __bfloat162float(tile[(b * 32 + j) * kPitch + c]);
        amax = fmaxf(amax, fabsf(v[j]));
      }
      const uint32_t e = e8m0_from_amax(amax);
      const float inv = inv_scale_from_e8m0(e);
      if (c0 + c < C) {
        uint32_t w[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = pack4_e4m3(v[4 * j] * inv, v[4 * j + 1] * inv, v[4 * j + 2] * inv, v[4 * j + 3] * inv);
        uint8_t* dst = qt + (long long)(c0 + c) * ldqt + r0 + b * 32;
        if (r0 + b * 32 + 32 <= R) {
          reinterpret_cast<uint4*>(dst)[0] = make_uint4(w[0], w[1], w[2], w[3]);
          reinterpret_cast<uint4*>(dst)[1] = make_uint4(w[4], w[5], w[6], w[7]);
        } else {
          for (int j = 0; j < 32; ++j)
            if (r0 + b * 32 + j < R) dst[j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
      }
      sft[((size_t)tc * sft_katoms + tr) * 512 + (c & 31) * 16 + (c >> 5) * 4 + b] = (uint8_t)e;
    }
  }
}

}  // namespace

// sf must hold ceil(R/128) x ceil(C/128) atoms of 512 bytes, sft ceil(C/128) x ceil(R/128); zero-initialised by the
// caller (the padding rows of the last atom are read by the GEMM's tiles).
cudaError_t quant_mxfp8(const void* x, long long ldx, int R, int C, void* q, long long ldq, void* sf, void* qt,
                        long long ldqt, void* sft, cudaStream_t stream) {
  if (R <= 0 || C <= 0) return cudaSuccess;
  if (ldx % 8 != 0 || (q && ldq % 16 != 0) || (qt && ldqt % 16 != 0)) return cudaErrorInvalidValue;
  // the kernel loads x and stores q / qt 16 bytes at a time
  const auto misaligned = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; };
  if (misaligned(x) || (q && misaligned(q)) || (qt && misaligned(qt))) return cudaErrorInvalidValue;
  dim3 grid((C + kTile - 1) / kTile, (R + kTile - 1) / kTile);
  quant_mxfp8_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*)x, ldx, R, C, (uint8_t*)q, ldq, (uint8_t*)sf,
                                               (C + kTile - 1) / kTile, (uint8_t*)qt, ldqt, (uint8_t*)sft,
                                               (R + kTile - 1) / kTile);
  return cudaGetLastError();
}

}  // namespace tb
