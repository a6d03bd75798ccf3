// Flash-attention entry points (csrc/attn/flash_fwd.cu, flash_bwd.cu).
// Tensors are token-major [tokens, heads, D] bf16 or fp16 (is_bf16) with an arbitrary token stride (so q/k/v may be column blocks of
// one fused QKV activation); sequences are either fixed length (B x S) or packed with int32 cu_seqlens [B+1].
// alibi_slopes: optional fp32 [Hq] (alibi_batch_stride == 0) or [B, Hq] (stride Hq): bias -slope * |i + Sk - Sq - j|.
#pragma once
#include <cuda_runtime.h>

namespace tb {

// Fixed-length batches only: sequence b starts at token b * q_bs + q_off (keys: b * k_bs + k_off) of the flat token
// space; a stride of 0 means "dense" (q_bs = Sq, k_bs = Sk).  Blockwise (ring) attention uses it to address the second
// half of every query sequence or one half of a K/V block in place.
struct BlockView {
  int q_bs = 0, q_off = 0, k_bs = 0, k_off = 0;
  // attention dropout (csrc/attn/dropout.cuh): probability and the 64-bit seed that keys the counter-based mask; the
  // backward must be called with the same values
  float p_drop = 0.f;
  unsigned long long seed = 0;
};

// Blockwise forward: with `acc` (fp32 [Tq, Hq, D]) the epilogue merges the block into the running (acc, lse) pair and
// writes the merged result to o; acc_init != 0 for the first block of a row range.
cudaError_t flash_attn_fwd_ex(const void* q, const void* k, const void* v, void* o, float* lse, const int* cu_q,
                              const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D, long long q_ts,
                              long long k_ts, long long v_ts, long long o_ts, float scale, bool causal, int wl, int wr,
                              long long Tq, long long Tk, int max_q_len, bool is_bf16, const float* alibi_slopes,
                              int alibi_batch_stride, BlockView view, float* acc, int acc_init, cudaStream_t stream);

// Blockwise backward: phases bit 0 = preprocess (delta = rowsum(dO o O), dq_acc = 0), bit 1 = main kernel (dK/dV of the
// visited keys, dQ reduce-added into dq_acc), bit 2 = dq = cast(dq_acc).  A ring step runs bit 1 only.
// deterministic: bit 0 computes delta only, bit 1 computes dK/dV only, bit 2 runs the query-stationary dQ kernel, which
// writes dq directly without atomics (bitwise reproducible; dq_acc is not used and may be null).
cudaError_t flash_attn_bwd_ex(const void* q, const void* k, const void* v, const void* o, const void* dout,
                              const float* lse, void* dq, void* dk, void* dv, float* dq_acc, float* delta,
                              const int* cu_q, const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D,
                              long long q_ts, long long k_ts, long long v_ts, long long do_ts, float scale, bool causal,
                              int wl, int wr, long long Tq, long long Tk, long long dq_ts, long long dk_ts,
                              long long dv_ts, int num_sms, bool is_bf16, const float* alibi_slopes,
                              int alibi_batch_stride, BlockView view, int phases, cudaStream_t stream,
                              bool deterministic = false);

cudaError_t flash_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const int* cu_q,
                           const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D, long long q_ts,
                           long long k_ts, long long v_ts, long long o_ts, float scale, bool causal, int wl, int wr,
                           long long Tq, long long Tk, int max_q_len, bool is_bf16, const float* alibi_slopes,
                           int alibi_batch_stride, cudaStream_t stream);

cudaError_t flash_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                           const float* lse, void* dq, void* dk, void* dv, float* dq_acc, float* delta,
                           const int* cu_q, const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D,
                           long long q_ts, long long k_ts, long long v_ts, long long do_ts, float scale, bool causal,
                           int wl, int wr, long long Tq, long long Tk, long long dq_ts, long long dk_ts,
                           long long dv_ts, int num_sms, bool is_bf16, const float* alibi_slopes,
                           int alibi_batch_stride, cudaStream_t stream);

// Debug: when non-null, CTA (0,0,0) of the backward kernel writes clock64() stamps [64 iterations][16 slots].
void flash_attn_bwd_set_trace(long long* p);
void flash_attn_fwd_set_trace(long long* p);

}  // namespace tb
