// (16-bit kernels take `is_bf16`: false = IEEE fp16 -- reference benchmarks run both, benchmarks/run.sh:8-48)
// C++ entry points of the bandwidth-bound op kernels (raw pointers + stream; wrapped by csrc/capi.cpp).
#pragma once
#include <cuda_runtime.h>

namespace tb {

cudaError_t rmsnorm_fwd(const void* x, const void* res, const void* w, void* y, void* h_out, float* rstd, int rows,
                        int H, float eps, int num_sms, bool is_bf16, cudaStream_t stream);
cudaError_t rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                        float* dw_partial, int dw_rows, int rows, int H, int num_sms, bool is_bf16,
                        cudaStream_t stream);
cudaError_t rope_inplace(void* x, const float* cos_t, const float* sin_t, const int* positions, long long T,
                         int nheads, int D, long long token_stride, int seq_len, bool backward, int num_sms,
                         bool is_bf16, cudaStream_t stream);
// Per-head RMSNorm of the q and k rows of a packed QKV buffer followed by RoPE, out of place (V rows copied); rstd is
// [T, hq + hk] fp32.  The backward writes dx and per-CTA weight-gradient partials dw_partial [dw_rows, 2, D] (q, k).
cudaError_t qk_norm_rope_fwd(const void* x, void* out, const void* q_weight, const void* k_weight, float* rstd,
                             const float* cos_t, const float* sin_t, const int* positions, long long T, int hq, int hk,
                             int D, long long token_stride, int seq_len, float eps, int num_sms, bool is_bf16,
                             cudaStream_t stream);
cudaError_t qk_norm_rope_bwd(const void* g, const void* x, void* dx, const void* q_weight, const void* k_weight,
                             const float* rstd, float* dw_partial, int dw_rows, const float* cos_t, const float* sin_t,
                             const int* positions, long long T, int hq, int hk, int D, long long token_stride,
                             int seq_len, int num_sms, bool is_bf16, cudaStream_t stream);
cudaError_t swiglu_fwd(const void* g, const void* u, void* h, long long T, int F, long long ldg, long long ldu,
                       int num_sms, bool is_bf16, cudaStream_t stream);
cudaError_t swiglu_bwd(const void* dh, const void* g, const void* u, void* dg, void* du, long long T, int F,
                       long long ldg, long long ldu, long long lddg, long long lddu, int num_sms, bool is_bf16,
                       cudaStream_t stream);
cudaError_t cross_entropy_fwd_bwd(void* logits, const long long* labels, float* loss_rows, float* lse_rows, int n,
                                  int V, long long ld, int ignore_index, const float* scale_ptr, float scale_val,
                                  bool write_grad, cudaStream_t stream);
// step counts every call; skipped (optional, int32 device counter) counts the calls that found_inf skipped.  With it
// the bias correction uses step - *skipped, computed on the device; without it, step (computed on the host).
cudaError_t adamw_flat(float* p, const void* g, bool grad_is_bf16, float* m, float* v, void* p_lp, long long n,
                       float lr, float beta1, float beta2, float eps, float weight_decay, int step, int* skipped,
                       const float* grad_scale, const float* found_inf, int num_sms, cudaStream_t stream);
cudaError_t sqnorm_accumulate(const void* g, bool is_bf16, long long n, float* out, float pre_scale, int num_sms,
                              cudaStream_t stream);
// Same sums in a fixed order (bitwise reproducible), one launch: partial = fp32 workspace of >= 8 * num_sms floats,
// counter = one zeroed uint32 that the launch leaves zeroed again; launches sharing them must be stream-ordered.
cudaError_t sqnorm_accumulate_ordered(const void* g, bool is_bf16, long long n, float* out, float pre_scale,
                                      float* partial, unsigned int* counter, int num_sms, cudaStream_t stream);
// MX-FP8 quantiser (ops/quant_mxfp8.cu): row-wise (q, sf) and / or transposed (qt, sft) e4m3 + UE8M0 outputs of a bf16
// matrix x[R][C]; either pair may be null.
cudaError_t quant_mxfp8(const void* x, long long ldx, int R, int C, void* q, long long ldq, void* sf, void* qt,
                        long long ldqt, void* sft, cudaStream_t stream);
// Mixture-of-experts routing (ops/moe.cu), deterministic: see the comment at the top of that file.
// Router: softmax over E <= 256 logits (dtype 0 = fp32, 1 = bf16, 2 = fp16), top-k <= 8, optional renormalisation of
// the k fp32 weights; the backward maps d(weights) to d(logits).
cudaError_t moe_router_fwd(const void* logits, float* weights, long long* ids, int T, int E, int k, bool norm,
                           int dtype, cudaStream_t stream);
cudaError_t moe_router_bwd(const void* logits, const long long* ids, const float* dweights, void* dlogits, int T, int E,
                           int k, bool norm, int dtype, cudaStream_t stream);
// Index build for ids [T*k]: counts [E], 128-row padded offsets [E+1], tile_expert [rows/128], *num_m_tiles, pos [T*k]
// (row of each entry, stable order inside an expert) and row_src [rows] (entry of each row, -1 for padding).
// rows >= T*k + E*127, rows % 128 == 0.
cudaError_t moe_index(const long long* ids, int T, int k, int E, int rows, int* counts, int* offsets, int* tile_expert,
                      int* num_m_tiles, int* pos, int* row_src, cudaStream_t stream);
cudaError_t moe_permute(const void* x, const int* row_src, const int* offsets, void* x_perm, int rows, int k, int E,
                        int H, int num_sms, cudaStream_t stream);
cudaError_t moe_unpermute_sum(const void* dx_perm, const int* pos, void* dx, int T, int k, int H, int num_sms,
                              bool is_bf16, cudaStream_t stream);
cudaError_t moe_combine_fwd(const void* y_perm, const int* pos, const float* w, const void* residual, void* out, int T,
                            int k, int H, int num_sms, bool is_bf16, cudaStream_t stream);
cudaError_t moe_combine_bwd(const void* dout, const void* y_perm, const int* row_src, const int* offsets, const float* w,
                            void* dy_perm, float* dw, int rows, int k, int E, int H, int num_sms, bool is_bf16,
                            cudaStream_t stream);
cudaError_t scale_inplace(void* g, bool is_bf16, long long n, const float* scale, int num_sms, cudaStream_t stream);

}  // namespace tb
