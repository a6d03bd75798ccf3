// Public (C++) entry points of the wgmma GEMM family.  Raw pointers + stream so the kernels build
// without any PyTorch headers; csrc/bindings.cpp wraps them as torch ops.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tb {

// D[M,N] (+)= A_op[M,K] * B_op[N,K]^T (+ bias).  bf16 (or, with is_fp16, IEEE fp16) inputs, fp32 accumulation in registers.
//   a_mn_major == false : A stored [M][K] (row pitch lda);  true : A stored [K][M]
//   b_mn_major == false : B stored [N][K] (row pitch ldb);  true : B stored [K][N]
//   out_fp32            : D is float32 instead of bf16
//   accumulate          : D += result (gradient accumulation)
//   cluster             : 1 or 2, kept for ABI compatibility: sm_90a has no CTA-pair MMA, every tile is 128x256 on one CTA
cudaError_t gemm_bf16(const void* A, const void* B, void* D, const void* bias, int M, int N, int K, long long lda,
                      long long ldb, long long ldd, bool a_mn_major, bool b_mn_major, bool out_fp32, bool accumulate,
                      int cluster, int num_sms, cudaStream_t stream, bool is_fp16 = false);

// Grid shape of the unfused GEMM: 0 = "static", a persistent grid striped over the tiles; 1 = "dynamic", a plain grid
// of one CTA per tile, so that SMs busy with a concurrent kernel simply receive fewer tiles.  mode < 0 queries.
int gemm_sched_mode(int mode);

// Same with a separate addend: D = A_op * B_op^T (+ bias) + C, C with D's dtype and row pitch ldc (C may alias D).
// Used to fuse the transformer residual add into the down-projection epilogue.
cudaError_t gemm_bf16_ex(const void* A, const void* B, void* D, const void* bias, const void* C, int M, int N, int K,
                         long long lda, long long ldb, long long ldd, long long ldc, bool a_mn_major, bool b_mn_major,
                         bool out_fp32, int cluster, int num_sms, cudaStream_t stream, bool is_fp16 = false);

// gate|up projection with the SwiGLU activation in the epilogue: H[M][F] = silu(A Wg^T) * (A Wu^T), W_gu = [Wg; Wu]
// stored [2F][K]; GU (optional, [M][2F]) receives the pre-activation for the backward pass.  F % 128 == 0.
cudaError_t gemm_swiglu_bf16(const void* A, const void* Wgu, void* H, void* GU, int M, int F, int K, long long lda,
                             long long ldb, long long ldh, long long ldgu, int num_sms, cudaStream_t stream,
                             bool is_fp16 = false);

// ---- grouped (mixture-of-experts) GEMMs over expert-sorted rows (see GroupArgs in gemm_bf16.cu) ----
// Rows of A are tokens sorted by expert, every expert's segment padded with zero rows to a multiple of 128; M is the
// padded row capacity (a multiple of 128).  tile_expert[m_tile] is the expert of each 128-row tile and *num_m_tiles
// the number of valid tiles; both stay on the device.
// D[M, N] = A[M, K] B_e^T: B is [E*N][K] (b_mn_major == false, forward) or [E*K][N] (true, dgrad: B_e read transposed).
cudaError_t gemm_grouped_bf16(const void* A, const void* B, void* D, int M, int N, int K, int E, long long lda,
                              long long ldb, long long ldd, bool b_mn_major, const int* tile_expert,
                              const int* num_m_tiles, int num_sms, cudaStream_t stream, bool is_fp16 = false);
// gate|up projection with the SwiGLU epilogue per expert: W_gu is [E*2F][K], expert e's gate rows start at e*2F and its
// up rows at e*2F + F.  F % 128 == 0.
cudaError_t gemm_grouped_swiglu_bf16(const void* A, const void* Wgu, void* H, void* GU, int M, int F, int K, int E,
                                     long long lda, long long ldb, long long ldh, long long ldgu,
                                     const int* tile_expert, const int* num_m_tiles, int num_sms, cudaStream_t stream,
                                     bool is_fp16 = false);
// wgrad: D[e*M : e*M + M, N] (+)= dY_e^T X_e, reducing over expert e's padded rows [offsets[e], offsets[e+1]) of
// dY [rows][M] and X [rows][N].  An expert without rows writes zeros (or leaves D unchanged when accumulating).
cudaError_t gemm_grouped_wgrad_bf16(const void* dY, const void* X, void* D, int M, int N, int E, int rows,
                                    long long lda, long long ldb, long long ldd, const int* offsets, bool out_fp32,
                                    bool accumulate, int num_sms, cudaStream_t stream, bool is_fp16 = false);

// ---- fused tensor-parallel kernels (see the FuseArgs comment in gemm_bf16.cu) ----
// all-gather -> GEMM: D[world*rows, N] = gather(A)[world*rows, K] * B_op^T.  `a_full` is this rank's symmetric
// gathered buffer whose own row block is already filled; `peer_a_full[r]` is rank r's mapping of the same buffer.
cudaError_t ag_gemm_bf16(const uint64_t* peer_a_full, const uint64_t* pad_ptrs, void* a_full, const void* B, void* D,
                         const void* bias, int rows_per_rank, int N, int K, long long ldb, long long ldd,
                         bool b_mn_major, int rank, int world, uint32_t* flags, uint32_t flag_target,
                         uint32_t* block_counter, int channel, uint32_t epoch, int comm_clusters, int num_sms,
                         cudaStream_t stream);
// GEMM -> reduce-scatter, part 1: partial tiles are stored into the owner rank's staging slot [rank] (peer stores)
// and counted in peer_counters[owner][rank] (8 arrivals per 128-row CTA tile: one per MMA warp).
cudaError_t gemm_rs_bf16(const void* A, const void* B, const uint64_t* peer_stage, const uint64_t* peer_counters,
                         const uint64_t* pad_ptrs, int rows_per_rank, int N, int K, long long lda, long long ldb,
                         bool a_mn_major, bool b_mn_major, int rank, int world, int channel, uint32_t epoch,
                         int num_sms, cudaStream_t stream);
// part 2: out = sum over sources of stage[src] (+ residual) once counters[src] >= expected for every source.
cudaError_t rs_reduce_bf16(const void* stage, const uint32_t* counters, uint32_t expected, const void* residual,
                           void* out, int rows, int N, int world, long long slot_stride, int num_sms, cudaStream_t stream);

// Block-scaled FP8 GEMM (gemm_mxfp8.cu): D[M,N] = (A[M,K] * SFA) (B[N,K] * SFB)^T (+ C); e4m3 operands, UE8M0 scales per
// 32 elements of K in the atom-tiled layout written by ops/quant_mxfp8.cu; K % 128 == 0.
cudaError_t gemm_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, const void* C, int M,
                       int N, int K, long long lda, long long ldb, long long ldd, long long ldc, bool out_fp32,
                       int num_sms, cudaStream_t stream);
// Grouped MX-FP8 GEMMs over expert-sorted rows (the layout of the grouped bf16 GEMMs above); bf16 output.
// Forward (b_transposed == false): B is [E*N][K] and N % 128 == 0.  Dgrad (true): B is [N][E*K], the transposed
// quantisation of an [E*K][N] weight.  M % 128 == 0, K % 128 == 0.
cudaError_t gemm_grouped_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, int M, int N,
                               int K, int E, long long lda, long long ldb, long long ldd, bool b_transposed,
                               const int* tile_expert, const int* num_m_tiles, int num_sms, cudaStream_t stream);
// wgrad: D[e*M : e*M + M, N] (+)= A_e B_e^T over expert e's padded rows [offsets[e], offsets[e+1]) of A [M][rows] and
// B [N][rows] (transposed quantisations, scales along the rows); D fp32 or bf16.  rows % 128 == 0.
cudaError_t gemm_grouped_wgrad_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, int M,
                                     int N, int E, int rows, long long lda, long long ldb, long long ldd,
                                     const int* offsets, bool out_fp32, bool accumulate, int num_sms,
                                     cudaStream_t stream);

}  // namespace tb
