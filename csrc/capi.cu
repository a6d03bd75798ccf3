// Flat C ABI over the native kernels, loaded from Python with ctypes (torchacc_b200/_native.py).
// Every function returns a cudaError_t as int; pointers are raw device addresses (tensor.data_ptr()) and
// `stream` is a cudaStream_t handle (torch.cuda.current_stream().cuda_stream).
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "attn/attn.h"
#include "comm/comm.h"
#include "gemm/gemm.h"
#include "ops/ops.h"

#define TB_API extern "C" __attribute__((visibility("default")))

static inline cudaStream_t S(uint64_t s) { return reinterpret_cast<cudaStream_t>(s); }
template <typename T>
static inline T* P(uint64_t p) { return reinterpret_cast<T*>(p); }

TB_API const char* tb_error_string(int code) { return cudaGetErrorString(static_cast<cudaError_t>(code)); }
TB_API int tb_abi_version() { return 5; }

TB_API int tb_device_info(int device, int* num_sms, int* cc_major, int* cc_minor, long long* smem_optin) {
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) return (int)e;
  *num_sms = prop.multiProcessorCount;
  *cc_major = prop.major;
  *cc_minor = prop.minor;
  *smem_optin = (long long)prop.sharedMemPerBlockOptin;
  return 0;
}

// ---- GEMM -------------------------------------------------------------------------------------------
TB_API int tb_gemm_bf16(uint64_t A, uint64_t B, uint64_t D, uint64_t bias, int M, int N, int K, long long lda,
                        long long ldb, long long ldd, int a_mn_major, int b_mn_major, int out_fp32, int accumulate,
                        int cluster, int num_sms, uint64_t stream, int is_fp16) {
  return (int)tb::gemm_bf16(P<void>(A), P<void>(B), P<void>(D), P<void>(bias), M, N, K, lda, ldb, ldd,
                            a_mn_major != 0, b_mn_major != 0, out_fp32 != 0, accumulate != 0, cluster, num_sms,
                            S(stream), is_fp16 != 0);
}

TB_API int tb_gemm_sched_mode(int mode) { return tb::gemm_sched_mode(mode); }
TB_API int tb_gemm_bf16_ex(uint64_t A, uint64_t B, uint64_t D, uint64_t bias, uint64_t C, int M, int N, int K,
                           long long lda, long long ldb, long long ldd, long long ldc, int a_mn_major, int b_mn_major,
                           int out_fp32, int cluster, int num_sms, uint64_t stream, int is_fp16) {
  return (int)tb::gemm_bf16_ex(P<void>(A), P<void>(B), P<void>(D), P<void>(bias), P<void>(C), M, N, K, lda, ldb, ldd, ldc,
                               a_mn_major != 0, b_mn_major != 0, out_fp32 != 0, cluster, num_sms, S(stream),
                               is_fp16 != 0);
}

// ---- norm / rope / activation -----------------------------------------------------------------------
TB_API int tb_rmsnorm_fwd(uint64_t x, uint64_t res, uint64_t w, uint64_t y, uint64_t h_out, uint64_t rstd, int rows,
                          int H, float eps, int num_sms, uint64_t stream, int is_bf16) {
  return (int)tb::rmsnorm_fwd(P<void>(x), P<void>(res), P<void>(w), P<void>(y), P<void>(h_out), P<float>(rstd), rows,
                              H, eps, num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_rmsnorm_bwd(uint64_t dy, uint64_t x, uint64_t w, uint64_t rstd, uint64_t dres, uint64_t dx, uint64_t dw,
                          int dw_rows, int rows, int H, int num_sms, uint64_t stream, int is_bf16) {
  return (int)tb::rmsnorm_bwd(P<void>(dy), P<void>(x), P<void>(w), P<float>(rstd), P<void>(dres), P<void>(dx),
                              P<float>(dw), dw_rows, rows, H, num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_rope_inplace(uint64_t x, uint64_t cos_t, uint64_t sin_t, uint64_t positions, long long T, int nheads,
                           int D, long long token_stride, int seq_len, int backward, int num_sms, uint64_t stream,
                           int is_bf16) {
  return (int)tb::rope_inplace(P<void>(x), P<float>(cos_t), P<float>(sin_t), P<int>(positions), T, nheads, D,
                               token_stride, seq_len, backward != 0, num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_qk_norm_rope_fwd(uint64_t x, uint64_t out, uint64_t q_weight, uint64_t k_weight, uint64_t rstd,
                               uint64_t cos_t, uint64_t sin_t, uint64_t positions, long long T, int hq, int hk, int D,
                               long long token_stride, int seq_len, float eps, int num_sms, uint64_t stream,
                               int is_bf16) {
  return (int)tb::qk_norm_rope_fwd(P<void>(x), P<void>(out), P<void>(q_weight), P<void>(k_weight), P<float>(rstd),
                                   P<float>(cos_t), P<float>(sin_t), P<int>(positions), T, hq, hk, D, token_stride,
                                   seq_len, eps, num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_qk_norm_rope_bwd(uint64_t g, uint64_t x, uint64_t dx, uint64_t q_weight, uint64_t k_weight,
                               uint64_t rstd, uint64_t dw_partial, int dw_rows, uint64_t cos_t, uint64_t sin_t,
                               uint64_t positions, long long T, int hq, int hk, int D, long long token_stride,
                               int seq_len, int num_sms, uint64_t stream, int is_bf16) {
  return (int)tb::qk_norm_rope_bwd(P<void>(g), P<void>(x), P<void>(dx), P<void>(q_weight), P<void>(k_weight),
                                   P<float>(rstd), P<float>(dw_partial), dw_rows, P<float>(cos_t), P<float>(sin_t),
                                   P<int>(positions), T, hq, hk, D, token_stride, seq_len, num_sms, is_bf16 != 0,
                                   S(stream));
}
TB_API int tb_swiglu_fwd(uint64_t g, uint64_t u, uint64_t h, long long T, int F, long long ldg, long long ldu,
                         int num_sms, uint64_t stream, int is_bf16) {
  return (int)tb::swiglu_fwd(P<void>(g), P<void>(u), P<void>(h), T, F, ldg, ldu, num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_swiglu_bwd(uint64_t dh, uint64_t g, uint64_t u, uint64_t dg, uint64_t du, long long T, int F,
                         long long ldg, long long ldu, long long lddg, long long lddu, int num_sms, uint64_t stream,
                         int is_bf16) {
  return (int)tb::swiglu_bwd(P<void>(dh), P<void>(g), P<void>(u), P<void>(dg), P<void>(du), T, F, ldg, ldu, lddg,
                             lddu, num_sms, is_bf16 != 0, S(stream));
}

// ---- loss / optimizer -------------------------------------------------------------------------------
TB_API int tb_cross_entropy(uint64_t logits, uint64_t labels, uint64_t loss_rows, uint64_t lse_rows, int n, int V,
                            long long ld, int ignore_index, uint64_t scale_ptr, float scale_val, int write_grad,
                            uint64_t stream) {
  return (int)tb::cross_entropy_fwd_bwd(P<void>(logits), P<long long>(labels), P<float>(loss_rows), P<float>(lse_rows),
                                        n, V, ld, ignore_index, P<float>(scale_ptr), scale_val, write_grad != 0,
                                        S(stream));
}
TB_API int tb_adamw_flat(uint64_t p, uint64_t g, int grad_is_bf16, uint64_t m, uint64_t v, uint64_t p_lp, long long n,
                         float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                         uint64_t skipped, uint64_t grad_scale, uint64_t found_inf, int num_sms, uint64_t stream) {
  return (int)tb::adamw_flat(P<float>(p), P<void>(g), grad_is_bf16 != 0, P<float>(m), P<float>(v), P<void>(p_lp), n,
                             lr, beta1, beta2, eps, weight_decay, step, P<int>(skipped), P<float>(grad_scale),
                             P<float>(found_inf), num_sms, S(stream));
}
TB_API int tb_sqnorm_accumulate(uint64_t g, int is_bf16, long long n, uint64_t out, float pre_scale, int num_sms,
                                uint64_t stream) {
  return (int)tb::sqnorm_accumulate(P<void>(g), is_bf16 != 0, n, P<float>(out), pre_scale, num_sms, S(stream));
}
TB_API int tb_sqnorm_accumulate_ordered(uint64_t g, int is_bf16, long long n, uint64_t out, float pre_scale,
                                        uint64_t partial, uint64_t counter, int num_sms, uint64_t stream) {
  return (int)tb::sqnorm_accumulate_ordered(P<void>(g), is_bf16 != 0, n, P<float>(out), pre_scale, P<float>(partial),
                                            P<unsigned int>(counter), num_sms, S(stream));
}
TB_API int tb_scale_inplace(uint64_t g, int is_bf16, long long n, uint64_t scale, int num_sms, uint64_t stream) {
  return (int)tb::scale_inplace(P<void>(g), is_bf16 != 0, n, P<float>(scale), num_sms, S(stream));
}

// ---- attention (csrc/attn/attn.h) ---------------------------------------------------------------------------
TB_API int tb_flash_attn_fwd(const tb::AttnParams* p, uint64_t stream) { return (int)tb::flash_attn_fwd(*p, S(stream)); }
TB_API int tb_flash_attn_bwd(const tb::AttnParams* p, int num_sms, uint64_t stream) {
  return (int)tb::flash_attn_bwd(*p, num_sms, S(stream));
}
TB_API long long tb_attn_bwd_set_profile(uint64_t buf, long long ctas) {
  return tb::attn_bwd_set_profile(P<unsigned long long>(buf), ctas);
}
// sizeof(AttnParams), then the offset of every field in declaration order, into out[0, n); returns the number of values
TB_API int tb_attn_params_layout(long long* out, int n) {
  using A = tb::AttnParams;
  const long long v[] = {
      sizeof(A),          offsetof(A, q),        offsetof(A, k),       offsetof(A, v),     offsetof(A, o),
      offsetof(A, dout),  offsetof(A, lse),      offsetof(A, dq),      offsetof(A, dk),    offsetof(A, dv),
      offsetof(A, dq_acc), offsetof(A, delta),   offsetof(A, q_ts),    offsetof(A, k_ts),  offsetof(A, v_ts),
      offsetof(A, o_ts),  offsetof(A, do_ts),    offsetof(A, dq_ts),   offsetof(A, dk_ts), offsetof(A, dv_ts),
      offsetof(A, cu_q),  offsetof(A, cu_k),     offsetof(A, B),       offsetof(A, Sq),    offsetof(A, Sk),
      offsetof(A, Hq),    offsetof(A, Hk),       offsetof(A, D),       offsetof(A, Tq),    offsetof(A, Tk),
      offsetof(A, scale), offsetof(A, causal),   offsetof(A, wl),      offsetof(A, wr),    offsetof(A, alibi),
      offsetof(A, alibi_bs), offsetof(A, p_drop), offsetof(A, seed),   offsetof(A, q_bs),  offsetof(A, q_off),
      offsetof(A, k_bs),  offsetof(A, k_off),    offsetof(A, acc),     offsetof(A, acc_init),
      offsetof(A, phases), offsetof(A, deterministic), offsetof(A, is_bf16)};
  const int total = (int)(sizeof(v) / sizeof(v[0]));
  for (int i = 0; i < n && i < total; ++i) out[i] = v[i];
  return total;
}

// ---- symmetric-memory communication ------------------------------------------------------------------------
TB_API int tb_symm_alloc(long long bytes, uint64_t* out_ptr) {
  void* p = nullptr;
  cudaError_t e = tb::symm_alloc((size_t)bytes, &p);
  *out_ptr = reinterpret_cast<uint64_t>(p);
  return (int)e;
}
TB_API int tb_symm_free(uint64_t ptr) { return (int)tb::symm_free(P<void>(ptr)); }
TB_API int tb_symm_get_handle(uint64_t ptr, void* handle64) { return (int)tb::symm_get_handle(P<void>(ptr), handle64); }
TB_API int tb_symm_open_handle(const void* handle64, uint64_t* out_ptr) {
  void* p = nullptr;
  cudaError_t e = tb::symm_open_handle(handle64, &p);
  *out_ptr = reinterpret_cast<uint64_t>(p);
  return (int)e;
}
TB_API int tb_symm_close_handle(uint64_t ptr) { return (int)tb::symm_close_handle(P<void>(ptr)); }
TB_API int tb_symm_all_gather(const uint64_t* peers, const uint64_t* pads, long long src_off, uint64_t out,
                              long long bytes, int rank, int world, int channel, uint32_t epoch, uint64_t counter,
                              int num_sms, uint64_t stream) {
  return (int)tb::symm_all_gather(peers, pads, (size_t)src_off, P<void>(out), (size_t)bytes, rank, world, channel, epoch,
                                  P<uint32_t>(counter), num_sms, S(stream));
}
TB_API int tb_symm_reduce_scatter(const uint64_t* peers, const uint64_t* pads, long long src_off, uint64_t out,
                                  long long n, int in_bf16, int out_fp32, float scale, int rank, int world, int channel,
                                  uint32_t epoch, uint64_t counter, int num_sms, uint64_t stream) {
  return (int)tb::symm_reduce_scatter(peers, pads, (size_t)src_off, P<void>(out), (size_t)n, in_bf16 != 0, out_fp32 != 0,
                                      scale, rank, world, channel, epoch, P<uint32_t>(counter), num_sms, S(stream));
}
TB_API int tb_symm_all_to_all(const uint64_t* peers, const uint64_t* pads, long long src_off, uint64_t out,
                              long long chunk_bytes, int rank, int world, int channel, uint32_t epoch, uint64_t counter,
                              int num_sms, uint64_t stream) {
  return (int)tb::symm_all_to_all(peers, pads, (size_t)src_off, P<void>(out), (size_t)chunk_bytes, rank, world, channel,
                                  epoch, P<uint32_t>(counter), num_sms, S(stream));
}

// ---- fused tensor-parallel GEMMs ---------------------------------------------------------------------------
TB_API int tb_ag_gemm_bf16(const uint64_t* peer_a_full, const uint64_t* pads, uint64_t a_full, uint64_t B, uint64_t D,
                           uint64_t bias, int rows_per_rank, int N, int K, long long ldb, long long ldd, int b_mn_major,
                           int rank, int world, uint64_t flags, uint32_t flag_target, uint64_t block_counter,
                           int channel, uint32_t epoch, int comm_clusters, int num_sms, uint64_t stream) {
  return (int)tb::ag_gemm_bf16(peer_a_full, pads, P<void>(a_full), P<void>(B), P<void>(D), P<void>(bias), rows_per_rank,
                               N, K, ldb, ldd, b_mn_major != 0, rank, world, P<uint32_t>(flags), flag_target,
                               P<uint32_t>(block_counter), channel, epoch, comm_clusters, num_sms, S(stream));
}
TB_API int tb_gemm_rs_bf16(uint64_t A, uint64_t B, const uint64_t* peer_stage, const uint64_t* peer_counters,
                           const uint64_t* pads, int rows_per_rank, int N, int K, long long lda, long long ldb,
                           int a_mn_major, int b_mn_major, int rank, int world, int channel, uint32_t epoch,
                           int num_sms, uint64_t stream) {
  return (int)tb::gemm_rs_bf16(P<void>(A), P<void>(B), peer_stage, peer_counters, pads, rows_per_rank, N, K, lda, ldb,
                               a_mn_major != 0, b_mn_major != 0, rank, world, channel, epoch, num_sms, S(stream));
}
TB_API int tb_rs_reduce_bf16(uint64_t stage, uint64_t counters, uint32_t expected, uint64_t residual, uint64_t out,
                             int rows, int N, int world, long long slot_stride, int num_sms, uint64_t stream) {
  return (int)tb::rs_reduce_bf16(P<void>(stage), P<uint32_t>(counters), expected, P<void>(residual), P<void>(out), rows,
                                 N, world, slot_stride, num_sms, S(stream));
}

// ---- collectives carried inside the GEMM kernels (csrc/fused/carry.*) ----------------------------------------
#include "fused/carry.h"
TB_API long long tb_carry_push(int kind, const uint64_t* src, uint64_t dst, const uint64_t* pads, long long bytes,
                               int rank, int world, int channel, uint32_t epoch, uint64_t block_counter, float scale,
                               int in_bf16, int out_fp32, int accumulate, uint64_t stats, int background,
                               int entry_channel, uint32_t entry_epoch) {
  return tb::carry_push(kind, src, dst, pads, bytes, rank, world, channel, epoch, block_counter, scale, in_bf16, out_fp32,
                        accumulate, stats, background, entry_channel, entry_epoch);
}
TB_API long long tb_carry_pending(long long job_id, int queue) { return tb::carry_pending(job_id, queue); }
TB_API int tb_carry_take_probe(double flops, long long* out8) { return tb::carry_take_probe(flops, out8); }
TB_API int tb_carry_flush(long long job_id, int queue, int num_sms, uint64_t stream) {
  return (int)tb::carry_flush(job_id, queue, num_sms, S(stream));
}
TB_API double tb_carry_bytes_per_flop(double v) { return tb::carry_bytes_per_flop(v); }
TB_API int tb_carry_stats(long long* out4, int reset) {
  tb::carry_stats(out4, reset);
  return 0;
}
TB_API int tb_symm_wait_done(const uint64_t* pads, int rank, int world, int channel, uint32_t epoch, uint64_t stream) {
  return (int)tb::symm_wait_done(pads, rank, world, channel, epoch, S(stream));
}
TB_API long long tb_carry_set_debug(uint64_t buf, long long records) {
  return tb::carry_set_debug(P<unsigned long long>(buf), records);
}
TB_API int tb_symm_signal(const uint64_t* pads, int rank, int world, int channel, uint32_t epoch, uint64_t stream) {
  return (int)tb::symm_signal(pads, rank, world, channel, epoch, S(stream));
}

// ---- block-scaled fp8 ---------------------------------------------------------------------------------------------
TB_API int tb_quant_mxfp8(uint64_t x, long long ldx, int R, int C, uint64_t q, long long ldq, uint64_t sf, uint64_t qt,
                          long long ldqt, uint64_t sft, uint64_t stream) {
  return (int)tb::quant_mxfp8(P<void>(x), ldx, R, C, P<void>(q), ldq, P<void>(sf), P<void>(qt), ldqt, P<void>(sft),
                              S(stream));
}
TB_API int tb_gemm_mxfp8(uint64_t A, uint64_t sfa, uint64_t B, uint64_t sfb, uint64_t D, uint64_t C, int M, int N, int K,
                         long long lda, long long ldb, long long ldd, long long ldc, int out_fp32, int num_sms,
                         uint64_t stream) {
  return (int)tb::gemm_mxfp8(P<void>(A), P<void>(sfa), P<void>(B), P<void>(sfb), P<void>(D), P<void>(C), M, N, K, lda, ldb,
                             ldd, ldc, out_fp32 != 0, num_sms, S(stream));
}
TB_API int tb_gemm_grouped_mxfp8(uint64_t A, uint64_t sfa, uint64_t B, uint64_t sfb, uint64_t D, int M, int N, int K,
                                 int E, long long lda, long long ldb, long long ldd, int b_transposed,
                                 uint64_t tile_expert, uint64_t num_m_tiles, int num_sms, uint64_t stream) {
  return (int)tb::gemm_grouped_mxfp8(P<void>(A), P<void>(sfa), P<void>(B), P<void>(sfb), P<void>(D), M, N, K, E, lda,
                                     ldb, ldd, b_transposed != 0, P<const int>(tile_expert),
                                     P<const int>(num_m_tiles), num_sms, S(stream));
}
TB_API int tb_gemm_grouped_wgrad_mxfp8(uint64_t A, uint64_t sfa, uint64_t B, uint64_t sfb, uint64_t D, int M, int N,
                                       int E, int rows, long long lda, long long ldb, long long ldd, uint64_t offsets,
                                       int out_fp32, int accumulate, int num_sms, uint64_t stream) {
  return (int)tb::gemm_grouped_wgrad_mxfp8(P<void>(A), P<void>(sfa), P<void>(B), P<void>(sfb), P<void>(D), M, N, E,
                                           rows, lda, ldb, ldd, P<const int>(offsets), out_fp32 != 0, accumulate != 0,
                                           num_sms, S(stream));
}
// ---- mixture of experts: grouped GEMMs (gemm/gemm_bf16.cu) and routing kernels (ops/moe.cu) --------------------
TB_API int tb_gemm_grouped(uint64_t A, uint64_t B, uint64_t D, int M, int N, int K, int E, long long lda, long long ldb,
                           long long ldd, int b_mn_major, uint64_t tile_expert, uint64_t num_m_tiles, int num_sms,
                           uint64_t stream, int is_fp16) {
  return (int)tb::gemm_grouped_bf16(P<void>(A), P<void>(B), P<void>(D), M, N, K, E, lda, ldb, ldd, b_mn_major != 0,
                                    P<const int>(tile_expert), P<const int>(num_m_tiles), num_sms, S(stream),
                                    is_fp16 != 0);
}
TB_API int tb_gemm_grouped_swiglu(uint64_t A, uint64_t Wgu, uint64_t H, uint64_t GU, int M, int F, int K, int E,
                                  long long lda, long long ldb, long long ldh, long long ldgu, uint64_t tile_expert,
                                  uint64_t num_m_tiles, int num_sms, uint64_t stream, int is_fp16) {
  return (int)tb::gemm_grouped_swiglu_bf16(P<void>(A), P<void>(Wgu), P<void>(H), P<void>(GU), M, F, K, E, lda, ldb, ldh,
                                           ldgu, P<const int>(tile_expert), P<const int>(num_m_tiles), num_sms,
                                           S(stream), is_fp16 != 0);
}
TB_API int tb_gemm_grouped_wgrad(uint64_t dY, uint64_t X, uint64_t D, int M, int N, int E, int rows, long long lda,
                                 long long ldb, long long ldd, uint64_t offsets, int out_fp32, int accumulate,
                                 int num_sms, uint64_t stream, int is_fp16) {
  return (int)tb::gemm_grouped_wgrad_bf16(P<void>(dY), P<void>(X), P<void>(D), M, N, E, rows, lda, ldb, ldd,
                                          P<const int>(offsets), out_fp32 != 0, accumulate != 0, num_sms, S(stream),
                                          is_fp16 != 0);
}
// router logits dtype: 0 = fp32, 1 = bf16, 2 = fp16
TB_API int tb_moe_router_fwd(uint64_t logits, uint64_t weights, uint64_t ids, int T, int E, int k, int norm_topk,
                             int dtype, uint64_t stream) {
  return (int)tb::moe_router_fwd(P<void>(logits), P<float>(weights), P<long long>(ids), T, E, k, norm_topk != 0, dtype,
                                 S(stream));
}
TB_API int tb_moe_router_bwd(uint64_t logits, uint64_t ids, uint64_t dweights, uint64_t dlogits, int T, int E, int k,
                             int norm_topk, int dtype, uint64_t stream) {
  return (int)tb::moe_router_bwd(P<void>(logits), P<long long>(ids), P<float>(dweights), P<void>(dlogits), T, E, k,
                                 norm_topk != 0, dtype, S(stream));
}
TB_API int tb_moe_index(uint64_t ids, int T, int k, int E, int rows, uint64_t counts, uint64_t offsets,
                        uint64_t tile_expert, uint64_t num_m_tiles, uint64_t pos, uint64_t row_src, uint64_t stream) {
  return (int)tb::moe_index(P<long long>(ids), T, k, E, rows, P<int>(counts), P<int>(offsets), P<int>(tile_expert),
                            P<int>(num_m_tiles), P<int>(pos), P<int>(row_src), S(stream));
}
TB_API int tb_moe_permute(uint64_t x, uint64_t row_src, uint64_t offsets, uint64_t x_perm, int rows, int k, int E, int H,
                          int num_sms, uint64_t stream) {
  return (int)tb::moe_permute(P<void>(x), P<int>(row_src), P<int>(offsets), P<void>(x_perm), rows, k, E, H, num_sms,
                              S(stream));
}
TB_API int tb_moe_unpermute_sum(uint64_t dx_perm, uint64_t pos, uint64_t dx, int T, int k, int H, int num_sms,
                                uint64_t stream, int is_bf16) {
  return (int)tb::moe_unpermute_sum(P<void>(dx_perm), P<int>(pos), P<void>(dx), T, k, H, num_sms, is_bf16 != 0,
                                    S(stream));
}
TB_API int tb_moe_combine_fwd(uint64_t y_perm, uint64_t pos, uint64_t w, uint64_t residual, uint64_t out, int T, int k,
                              int H, int num_sms, uint64_t stream, int is_bf16) {
  return (int)tb::moe_combine_fwd(P<void>(y_perm), P<int>(pos), P<float>(w), P<void>(residual), P<void>(out), T, k, H,
                                  num_sms, is_bf16 != 0, S(stream));
}
TB_API int tb_moe_combine_bwd(uint64_t dout, uint64_t y_perm, uint64_t row_src, uint64_t offsets, uint64_t w,
                              uint64_t dy_perm, uint64_t dw, int rows, int k, int E, int H, int num_sms,
                              uint64_t stream, int is_bf16) {
  return (int)tb::moe_combine_bwd(P<void>(dout), P<void>(y_perm), P<int>(row_src), P<int>(offsets), P<float>(w),
                                  P<void>(dy_perm), P<float>(dw), rows, k, E, H, num_sms, is_bf16 != 0, S(stream));
}

TB_API int tb_gemm_swiglu(uint64_t A, uint64_t Wgu, uint64_t H, uint64_t GU, int M, int F, int K, long long lda,
                          long long ldb, long long ldh, long long ldgu, int num_sms, uint64_t stream, int is_fp16) {
  return (int)tb::gemm_swiglu_bf16(P<void>(A), P<void>(Wgu), P<void>(H), P<void>(GU), M, F, K, lda, ldb, ldh, ldgu, num_sms,
                                   S(stream), is_fp16 != 0);
}
