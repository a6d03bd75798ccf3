// Stand-alone correctness + throughput harness for the wgmma GEMM (no PyTorch).
//   numerics : every (A-major, B-major, cluster, out dtype, accumulate, bias) combination against cuBLAS fp32-accum
//   perf     : Llama-3-8B shapes at T=8192 tokens, CUDA-event timed, L2 flushed between iterations,
//              next to cublasGemmEx on the same buffers.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O3 csrc/tests/gemm_test.cu csrc/gemm/gemm_bf16.cu -lcublas
#include <cublas_v2.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../gemm/gemm.h"

#define CK(x)                                                                          \
  do {                                                                                 \
    cudaError_t e_ = (x);                                                              \
    if (e_ != cudaSuccess) {                                                           \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);  \
      exit(2);                                                                         \
    }                                                                                  \
  } while (0)

__global__ void fill_kernel(__nv_bfloat16* p, size_t n, uint32_t seed, float scale) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t x = (uint32_t)i * 2654435761u + seed;
  x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;
  p[i] = __float2bfloat16(((x & 0xffff) / 65536.f - 0.5f) * scale);
}
__global__ void fill_f32(float* p, size_t n, float v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
// Naive fp32 reference: D[m,n] = sum_k A_op[m,k] * B_op[n,k]
__global__ void ref_kernel(const __nv_bfloat16* A, const __nv_bfloat16* B, float* D, int M, int N, int K, long lda,
                           long ldb, int a_mn, int b_mn) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  int m = blockIdx.y;
  if (n >= N) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) {
    float a = __bfloat162float(a_mn ? A[(long)k * lda + m] : A[(long)m * lda + k]);
    float b = __bfloat162float(b_mn ? B[(long)k * ldb + n] : B[(long)n * ldb + k]);
    acc += a * b;
  }
  D[(long)m * N + n] = acc;
}

static int num_sms = 132;
static int cl_mask = 3;  // bit0: cluster 1 kernels, bit1: cluster 2 kernels

static bool check_case(int M, int N, int K, int a_mn, int b_mn, int cluster, int out_fp32, int accumulate, int use_bias) {
  long lda = a_mn ? M : K, ldb = b_mn ? N : K;
  __nv_bfloat16 *A, *B, *bias;
  float* ref;
  void* D;
  size_t na = (size_t)M * K, nb = (size_t)N * K, nd = (size_t)M * N;
  CK(cudaMalloc(&A, na * 2)); CK(cudaMalloc(&B, nb * 2)); CK(cudaMalloc(&bias, N * 2));
  CK(cudaMalloc(&ref, nd * 4)); CK(cudaMalloc(&D, nd * 4));
  fill_kernel<<<(na + 255) / 256, 256>>>(A, na, 1u, 2.f);
  fill_kernel<<<(nb + 255) / 256, 256>>>(B, nb, 77u, 2.f);
  fill_kernel<<<(N + 255) / 256, 256>>>(bias, N, 5u, 4.f);
  // initial D contents (for accumulate): 0.5 (exact in bf16)
  if (out_fp32) fill_f32<<<(nd + 255) / 256, 256>>>((float*)D, nd, 0.5f);
  else {
    std::vector<__nv_bfloat16> h(nd, __float2bfloat16(0.5f));
    CK(cudaMemcpy(D, h.data(), nd * 2, cudaMemcpyHostToDevice));
  }
  ref_kernel<<<dim3((N + 127) / 128, M), 128>>>(A, B, ref, M, N, K, lda, ldb, a_mn, b_mn);
  CK(cudaGetLastError());
  cudaError_t e = tb::gemm_bf16(A, B, D, use_bias ? bias : nullptr, M, N, K, lda, ldb, N, a_mn, b_mn, out_fp32,
                                accumulate, cluster, num_sms, 0);
  if (e != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(e)); return false; }
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("kernel failed: %s\n", cudaGetErrorString(e)); exit(3); }
  std::vector<float> href(nd), hd(nd);
  std::vector<__nv_bfloat16> hb(nd), hbias(N);
  CK(cudaMemcpy(href.data(), ref, nd * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hbias.data(), bias, N * 2, cudaMemcpyDeviceToHost));
  if (out_fp32) CK(cudaMemcpy(hd.data(), D, nd * 4, cudaMemcpyDeviceToHost));
  else {
    CK(cudaMemcpy(hb.data(), D, nd * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < nd; ++i) hd[i] = __bfloat162float(hb[i]);
  }
  double max_err = 0, max_ref = 0;
  size_t bad = 0;
  for (size_t i = 0; i < nd; ++i) {
    float r = href[i] + (accumulate ? 0.5f : 0.f) + (use_bias ? __bfloat162float(hbias[i % N]) : 0.f);
    double err = fabs((double)hd[i] - r);
    double tol = (out_fp32 ? 2e-3 : 1e-2) * fmax(1.0, fabs((double)r)) + 1e-3 * sqrt((double)K);
    if (err > tol) ++bad;
    if (err > max_err) max_err = err;
    if (fabs(r) > max_ref) max_ref = fabs(r);
  }
  printf("  M=%d N=%d K=%d a_mn=%d b_mn=%d cl=%d f32=%d acc=%d bias=%d : max_err=%.4g (max|ref|=%.3g) bad=%zu %s\n", M, N,
         K, a_mn, b_mn, cluster, out_fp32, accumulate, use_bias, max_err, max_ref, bad, bad ? "FAIL" : "ok");
  cudaFree(A); cudaFree(B); cudaFree(bias); cudaFree(ref); cudaFree(D);
  return bad == 0;
}

static void perf_case(cublasHandle_t h, const char* name, int M, int N, int K, int a_mn, int b_mn, int iters) {
  long lda = a_mn ? M : K, ldb = b_mn ? N : K;
  __nv_bfloat16 *A, *B, *D;
  CK(cudaMalloc(&A, (size_t)M * K * 2)); CK(cudaMalloc(&B, (size_t)N * K * 2)); CK(cudaMalloc(&D, (size_t)M * N * 2));
  fill_kernel<<<((size_t)M * K + 255) / 256, 256>>>(A, (size_t)M * K, 1u, 1.f);
  fill_kernel<<<((size_t)N * K + 255) / 256, 256>>>(B, (size_t)N * K, 3u, 1.f);
  size_t flush_bytes = 256u << 20;
  void* flush;
  CK(cudaMalloc(&flush, flush_bytes));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  double flops = 2.0 * M * N * K;
  float alpha = 1.f, beta = 0.f;
  for (int mode = 0; mode < 4; ++mode) {  // 0: ours cluster1, 1: ours cluster2 (dynamic), 2: cuBLAS, 3: cluster2 static
    if (mode < 2 && !(cl_mask & (1 << mode))) continue;
    if (mode == 3 && !(cl_mask & 2)) continue;
    tb::gemm_sched_mode(mode == 3 ? 0 : 1);
    float best = 1e30f, total = 0;
    for (int i = 0; i < iters + 3; ++i) {
      CK(cudaMemsetAsync(flush, i, flush_bytes, 0));  // flush L2 (50 MB) between timed iterations
      cudaEventRecord(e0, 0);
      if (mode != 2) {
        cudaError_t e = tb::gemm_bf16(A, B, D, nullptr, M, N, K, lda, ldb, N, a_mn, b_mn, false, false,
                                      mode == 0 ? 1 : 2, num_sms, 0);
        if (e != cudaSuccess) { printf("launch failed %s\n", cudaGetErrorString(e)); exit(2); }
      } else {
        // row-major D[M,N] = A_op B_op^T  <=> column-major D^T[N,M] = B_op(cm) * A_op(cm)
        cublasOperation_t opB = b_mn ? CUBLAS_OP_N : CUBLAS_OP_T;  // first operand (B)
        cublasOperation_t opA = a_mn ? CUBLAS_OP_T : CUBLAS_OP_N;  // second operand (A)
        cublasStatus_t st = cublasGemmEx(h, opB, opA, N, M, K, &alpha, B, CUDA_R_16BF, (int)ldb, A, CUDA_R_16BF,
                                         (int)lda, &beta, D, CUDA_R_16BF, N, CUBLAS_COMPUTE_32F, CUBLAS_GEMM_DEFAULT);
        if (st != CUBLAS_STATUS_SUCCESS) { printf("cublas failed %d\n", (int)st); exit(2); }
      }
      cudaEventRecord(e1, 0);
      CK(cudaEventSynchronize(e1));
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (i >= 3) { total += ms; if (ms < best) best = ms; }
    }
    const char* mn = mode == 0 ? "tb cluster1" : mode == 1 ? "tb cl2 dyn " : mode == 2 ? "cuBLAS     " : "tb cl2 stat";
    printf("  %-10s %s M=%d N=%d K=%d : best %.3f ms (%.1f TFLOP/s)  mean %.3f ms (%.1f TFLOP/s)\n", name, mn, M, N, K,
           best, flops / best * 1e-9, total / iters, flops / (total / iters) * 1e-9);
  }
  tb::gemm_sched_mode(1);
  cudaFree(A); cudaFree(B); cudaFree(D); cudaFree(flush);
}

int main(int argc, char** argv) {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  num_sms = prop.multiProcessorCount;
  printf("device %s, %d SMs, cc %d.%d\n", prop.name, num_sms, prop.major, prop.minor);
  if (argc > 1) cl_mask = atoi(argv[1]);
  bool do_perf = argc < 3 || atoi(argv[2]) != 0;
  bool do_num = argc < 4 || atoi(argv[3]) != 0;
  bool ok = true;
  printf("== numerics ==\n");
  for (int cl = 1; cl <= 2 && do_num; ++cl)
    for (int a_mn = 0; a_mn < 2 && (cl_mask & cl); ++a_mn)
      for (int b_mn = 0; b_mn < 2; ++b_mn) {
        ok &= check_case(512, 512, 256, a_mn, b_mn, cl, 0, 0, 0);
        ok &= check_case(384, 768, 1024, a_mn, b_mn, cl, 1, 1, 0);
      }
  // ragged shapes (partial tiles in M, N and K), bias, bf16 accumulate
  for (int cl = 1; cl <= 2 && do_num; ++cl) {
    if (!(cl_mask & cl)) continue;
    ok &= check_case(200, 328, 136, 0, 0, cl, 0, 0, 1);
    ok &= check_case(200, 328, 136, 0, 1, cl, 1, 0, 0);
    ok &= check_case(200, 328, 136, 1, 1, cl, 0, 1, 1);
    ok &= check_case(4096, 1024, 512, 0, 0, cl, 0, 0, 0);  // several tiles per CTA: ring stage reuse
    ok &= check_case(2048, 2560, 192, 1, 1, cl, 0, 0, 0);
  }
  printf("numerics: %s\n", ok ? "ALL OK" : "FAILURES");
  if (do_perf) {
    cublasHandle_t h;
    cublasCreate(&h);
    printf("== perf (T=8192 tokens, Llama-3-8B) ==\n");
    const int T = 8192;
    perf_case(h, "fwd qkv", T, 6144, 4096, 0, 0, 10);
    perf_case(h, "fwd o", T, 4096, 4096, 0, 0, 10);
    perf_case(h, "fwd gateup", T, 28672, 4096, 0, 0, 10);
    perf_case(h, "fwd down", T, 4096, 14336, 0, 0, 10);
    perf_case(h, "dgrad gateup", T, 4096, 28672, 0, 1, 10);
    perf_case(h, "dgrad down", T, 14336, 4096, 0, 1, 10);
    perf_case(h, "wgrad gateup", 28672, 4096, T, 1, 1, 10);
    perf_case(h, "wgrad down", 4096, 14336, T, 1, 1, 10);
    perf_case(h, "square 8k", 8192, 8192, 8192, 0, 0, 10);
  }
  return ok ? 0 : 1;
}
