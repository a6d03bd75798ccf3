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
cudaError_t swiglu_fwd(const void* g, const void* u, void* h, long long T, int F, long long ldg, long long ldu,
                       int num_sms, bool is_bf16, cudaStream_t stream);
cudaError_t swiglu_bwd(const void* dh, const void* g, const void* u, void* dg, void* du, long long T, int F,
                       long long ldg, long long ldu, long long lddg, long long lddu, int num_sms, bool is_bf16,
                       cudaStream_t stream);
cudaError_t cross_entropy_fwd_bwd(void* logits, const long long* labels, float* loss_rows, float* lse_rows, int n,
                                  int V, long long ld, int ignore_index, const float* scale_ptr, float scale_val,
                                  bool write_grad, cudaStream_t stream);
cudaError_t adamw_flat(float* p, const void* g, bool grad_is_bf16, float* m, float* v, void* p_lp, long long n,
                       float lr, float beta1, float beta2, float eps, float weight_decay, int step,
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
cudaError_t scale_inplace(void* g, bool is_bf16, long long n, const float* scale, int num_sms, cudaStream_t stream);

}  // namespace tb
