// Problem description shared by the attention kernels (flash_fwd.cu, flash_bwd.cu) and the host code that fills it
// from an AttnParams.
#pragma once
#include <stdint.h>

#include "../common/tensormap.h"
#include "attn.h"
#include "dropout.cuh"

namespace tb {

// Kernel-side part of AttnParams that every attention kernel reads; the kernels' argument structs derive from it.
struct AttnShape {
  const int* cu_q;
  const int* cu_k;
  int B, Sq, Sk, Hq, Hk;
  long long Tq;
  float scale_log2, scale;
  int wl, wr;                     // visible keys of query position i: [i - wl, i + wr], < 0: unbounded; causal folded in
  const float* alibi;             // optional ALiBi slopes [Hq] (alibi_bs == 0) or [B, Hq]
  int alibi_bs;
  int q_bs, q_off, k_bs, k_off;   // fixed-length addressing (AttnParams), strides resolved
  DropoutParams drop;             // used by the kDrop instantiations only
};

// first token and length of query and key sequence b
__device__ __forceinline__ void seq_bounds(const AttnShape& s, int b, int& q_start, int& q_len, int& k_start,
                                           int& k_len) {
  q_start = s.cu_q ? s.cu_q[b] : b * s.q_bs + s.q_off;
  q_len = s.cu_q ? (s.cu_q[b + 1] - q_start) : s.Sq;
  k_start = s.cu_k ? s.cu_k[b] : b * s.k_bs + s.k_off;
  k_len = s.cu_k ? (s.cu_k[b + 1] - k_start) : s.Sk;
}

// Validates what both directions support (D in {64, 128}, Hq a multiple of Hk, p_drop < 1) and fills s from p.
inline cudaError_t make_shape(const AttnParams& p, AttnShape& s) {
  if (p.D != 64 && p.D != 128) return cudaErrorInvalidValue;
  if (p.Hq % p.Hk != 0) return cudaErrorInvalidValue;
  if (p.p_drop > 0.f && p.p_drop >= 1.f) return cudaErrorInvalidValue;
  s.cu_q = p.cu_q;
  s.cu_k = p.cu_k;
  s.B = p.B; s.Sq = p.Sq; s.Sk = p.Sk; s.Hq = p.Hq; s.Hk = p.Hk;
  s.Tq = p.Tq;
  s.scale = p.scale;
  s.scale_log2 = p.scale * 1.4426950408889634f;
  s.wl = p.wl;
  // causal caps the right bound at the diagonal: min(wr, 0) with an unbounded wr counted as +inf, which is 0 for every
  // wr (ops/attention.py::_mask_for applies the same rule)
  s.wr = p.causal ? 0 : p.wr;
  s.alibi = p.alibi;
  s.alibi_bs = p.alibi_bs;
  s.q_bs = p.q_bs > 0 ? p.q_bs : p.Sq; s.q_off = p.q_off;
  s.k_bs = p.k_bs > 0 ? p.k_bs : p.Sk; s.k_off = p.k_off;
  s.drop = DropoutParams{0u, 1.f, 0u, 0u};
  if (p.p_drop > 0.f) {
    s.drop.thresh24 = (uint32_t)((double)p.p_drop * 16777216.0 + 0.5);   // mirrored in dropout_keep_mask
    s.drop.rp = 1.f / (1.f - p.p_drop);
    s.drop.seed_lo = (uint32_t)(p.seed & 0xffffffffull);
    s.drop.seed_hi = (uint32_t)(p.seed >> 32);
  }
  return cudaSuccess;
}

// 3-D tensor map over a token-major [tokens, heads, D] bf16 / fp16 tensor with token stride `ts` elements:
// SWIZZLE_128B boxes of 64 columns x 1 head x `rows` tokens.
inline CUtensorMap make_map_thd(const void* base, long long tokens, int heads, int D, long long ts, bool bf16,
                                int rows) {
  uint64_t dims[3] = {(uint64_t)D, (uint64_t)heads, (uint64_t)tokens};
  uint64_t strides[2] = {(uint64_t)D * 2, (uint64_t)ts * 2};
  uint32_t box[3] = {64, 1, (uint32_t)rows};
  return make_tensor_map(base, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, dims,
                         strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace tb
