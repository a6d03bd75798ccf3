// Flash-attention entry points (csrc/attn/flash_fwd.cu, flash_bwd.cu).
// Tensors are token-major [tokens, heads, D] bf16 or fp16 (is_bf16) with an arbitrary token stride (so q/k/v may be column blocks of
// one fused QKV activation); sequences are either fixed length (B x S) or packed with int32 cu_seqlens [B+1].
// alibi: optional fp32 slopes [Hq] (alibi_bs == 0) or [B, Hq] (alibi_bs == Hq): bias -slope * |i + Sk - Sq - j|.
#pragma once
#include <cuda_runtime.h>

namespace tb {

// One attention call, forward or backward.  Mirrored field for field by a ctypes.Structure in
// torchacc_b200/ops/attention.py; tb_attn_params_layout (csrc/capi.cu) reports the layout so a test can compare them.
struct AttnParams {
  // token-major [tokens, heads, D] tensors and their token strides in elements; dout .. delta: backward only
  const void *q, *k, *v;
  void* o;
  const void* dout;
  float* lse;                           // [Hq, Tq]
  void *dq, *dk, *dv;
  float* dq_acc;                        // fp32 [Tq, Hq, D] dQ accumulator of the default backward
  float* delta;                         // fp32 [Hq, Tq] rowsum(dO o O)
  long long q_ts, k_ts, v_ts, o_ts, do_ts, dq_ts, dk_ts, dv_ts;
  const int *cu_q, *cu_k;               // null: fixed length
  int B, Sq, Sk, Hq, Hk, D;
  long long Tq, Tk;
  float scale;
  int causal, wl, wr;                   // bottom-right causal; window (left, right), < 0: unbounded
  const float* alibi;
  int alibi_bs;
  // attention dropout (csrc/attn/dropout.cuh): probability and the 64-bit seed that keys the counter-based mask; the
  // backward must be called with the same values
  float p_drop;
  unsigned long long seed;
  // fixed-length batches only: sequence b starts at token b * q_bs + q_off (keys: b * k_bs + k_off) of the flat token
  // space; a stride of 0 means "dense" (q_bs = Sq, k_bs = Sk).  Blockwise (ring) attention uses it to address the
  // second half of every query sequence or one half of a K/V block in place.
  int q_bs, q_off, k_bs, k_off;
  // blockwise forward: with `acc` (fp32 [Tq, Hq, D]) the epilogue merges the block into the running (acc, lse) pair and
  // writes the merged result to o; acc_init != 0 for the first block of a row range
  float* acc;
  int acc_init;
  // backward phases: bit 0 = preprocess (delta = rowsum(dO o O), dq_acc = 0), bit 1 = main kernel (dK/dV of the
  // visited keys, dQ reduce-added into dq_acc), bit 2 = dq = cast(dq_acc); 7 runs all three, a ring step bit 1 only.
  // deterministic: bit 0 computes delta only, bit 1 computes dK/dV only, bit 2 runs the query-stationary dQ kernel,
  // which writes dq directly without atomics (bitwise reproducible; dq_acc is not used and may be null).
  int phases, deterministic;
  int is_bf16;
};

cudaError_t flash_attn_fwd(const AttnParams& p, cudaStream_t stream);
cudaError_t flash_attn_bwd(const AttnParams& p, int num_sms, cudaStream_t stream);
// Phase profile of the head-dim-64 bf16 backward main kernel (benchmarks/attn_bwd_phases.py): while buf is set, that
// kernel runs an instrumented build that writes clock64() stamps of key tiles [0, ctas) of kv head 0, sequence 0 into
// buf (ctas records; layout in flash_bwd.cu at kProfHead).  Null turns it off.  Returns the u64 words per record.
long long attn_bwd_set_profile(unsigned long long* buf, long long ctas);

}  // namespace tb
