// Stand-alone correctness + throughput harness for the wgmma GEMM (no PyTorch).
//   numerics : every (A-major, B-major, cluster, out dtype, accumulate, bias) combination against cuBLAS fp32-accum
//   perf     : Llama-3-8B shapes and the GEMMs of one bench.py step at T=8192 tokens, CUDA-event timed, L2 flushed
//              between iterations; static and dynamic tile scheduling and cublasGemmEx on the same buffers.
//   fit      : per step shape (M, N), static scheduling and cuBLAS at K = 1024 ... 8192; a least-squares line through
//              time per round of tiles (ceil(tiles / SMs)) against K blocks of 64 separates the mainloop cost (slope)
//              from the fixed cost of a tile (intercept).
// Usage: gemm_test [cluster mask of the numerics: 1, 2 or 3] [perf 0|1] [numerics 0|1] [fit 0|1]
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O3 -I csrc csrc/tests/gemm_test.cu
//        csrc/gemm/gemm_bf16.cu csrc/fused/carry.cu -lcublas
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

// One shape, three implementations: our kernel under static and under dynamic tile scheduling, and cuBLAS.
// out_fp32 / accumulate as in the wgrad into an fp32 gradient buffer; d_off: elements between the allocation and D
// (the flat FSDP gradient keeps each weight at a multiple of 8 elements); addend: a residual C != D of D's shape added
// in the epilogue (cuBLAS: beta = 1 on D, the same bytes read); swiglu: the gate|up projection with its SwiGLU
// epilogue (N = 2F; always static; cuBLAS computes the plain GEMM).  Returns the mean times (ms) of the modes in
// `modes` (bit m: mode m).
struct PerfResult { float mean[3]; };
static PerfResult perf_case(cublasHandle_t h, const char* name, int M, int N, int K, int a_mn, int b_mn, int iters,
                            int out_fp32 = 0, int accumulate = 0, int swiglu = 0, int addend = 0, int d_off = 0,
                            int modes = 7) {
  PerfResult res = {{0.f, 0.f, 0.f}};
  long lda = a_mn ? M : K, ldb = b_mn ? N : K;
  __nv_bfloat16 *A, *B;
  void *Dalloc, *C = nullptr;
  const int esz = out_fp32 ? 4 : 2;
  const size_t dbytes = ((size_t)M * N + d_off) * esz;
  CK(cudaMalloc(&A, (size_t)M * K * 2)); CK(cudaMalloc(&B, (size_t)N * K * 2)); CK(cudaMalloc(&Dalloc, dbytes));
  CK(cudaMemset(Dalloc, 0, dbytes));
  void* D = (char*)Dalloc + (size_t)d_off * esz;
  if (addend) {
    CK(cudaMalloc(&C, (size_t)M * N * esz));
    CK(cudaMemset(C, 0, (size_t)M * N * esz));
  }
  fill_kernel<<<((size_t)M * K + 255) / 256, 256>>>(A, (size_t)M * K, 1u, 1.f);
  fill_kernel<<<((size_t)N * K + 255) / 256, 256>>>(B, (size_t)N * K, 3u, 1.f);
  size_t flush_bytes = 256u << 20;
  void* flush;
  CK(cudaMalloc(&flush, flush_bytes));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  double flops = 2.0 * M * N * K;
  float alpha = 1.f, beta = accumulate ? 1.f : 0.f;
  if (addend) beta = 1.f;
  for (int mode = 0; mode < 3; ++mode) {  // 0: ours, static; 1: ours, dynamic; 2: cuBLAS
    if (!(modes & (1 << mode))) continue;
    tb::gemm_sched_mode(mode == 1 ? 1 : 0);
    float best = 1e30f, total = 0;
    for (int i = 0; i < iters + 3; ++i) {
      CK(cudaMemsetAsync(flush, i, flush_bytes, 0));  // flush L2 (50 MB) between timed iterations
      cudaEventRecord(e0, 0);
      if (mode != 2) {
        cudaError_t e = swiglu ? tb::gemm_swiglu_bf16(A, B, D, nullptr, M, N / 2, K, lda, ldb, N / 2, 0, num_sms, 0)
                     : addend ? tb::gemm_bf16_ex(A, B, D, nullptr, C, M, N, K, lda, ldb, N, N, a_mn, b_mn, out_fp32,
                                                 1, num_sms, 0)
                              : tb::gemm_bf16(A, B, D, nullptr, M, N, K, lda, ldb, N, a_mn, b_mn, out_fp32,
                                              accumulate, 1, num_sms, 0);
        if (e != cudaSuccess) { printf("launch failed %s\n", cudaGetErrorString(e)); exit(2); }
      } else {
        // row-major D[M,N] = A_op B_op^T  <=> column-major D^T[N,M] = B_op(cm) * A_op(cm)
        cublasOperation_t opB = b_mn ? CUBLAS_OP_N : CUBLAS_OP_T;  // first operand (B)
        cublasOperation_t opA = a_mn ? CUBLAS_OP_T : CUBLAS_OP_N;  // second operand (A)
        cublasStatus_t st = cublasGemmEx(h, opB, opA, N, M, K, &alpha, B, CUDA_R_16BF, (int)ldb, A, CUDA_R_16BF,
                                         (int)lda, &beta, D, out_fp32 ? CUDA_R_32F : CUDA_R_16BF, N, CUBLAS_COMPUTE_32F,
                                         CUBLAS_GEMM_DEFAULT);
        if (st != CUBLAS_STATUS_SUCCESS) { printf("cublas failed %d\n", (int)st); exit(2); }
      }
      cudaEventRecord(e1, 0);
      CK(cudaEventSynchronize(e1));
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (i >= 3) { total += ms; if (ms < best) best = ms; }
    }
    const char* mn = mode == 0 ? "tb stat" : mode == 1 ? "tb dyn " : "cuBLAS ";
    printf("  %-14s %s M=%6d N=%6d K=%6d : best %7.3f ms (%5.1f TFLOP/s)  mean %7.3f ms (%5.1f TFLOP/s)\n", name, mn, M,
           N, K, best, flops / best * 1e-9, total / iters, flops / (total / iters) * 1e-9);
    res.mean[mode] = total / iters;
  }
  tb::gemm_sched_mode(0);
  cudaFree(A); cudaFree(B); cudaFree(Dalloc); cudaFree(C); cudaFree(flush);
  return res;
}

// the GEMMs of one bench.py step (Llama-3.2-1B: hidden 2048, 32/8 heads of 64, MLP 8192, vocab 128256, 16 layers;
// 2 x 4096 tokens, gradient checkpointing runs every forward GEMM twice, LM head in 4096-token chunks).  The o and
// down projections add the residual in their epilogue; the wgrads write into the fp32 flat gradient at an offset of
// 8 elements; the LM-head dW accumulates over its chunks.
struct Shape { const char* name; int M, N, K, a_mn, b_mn, f32, acc, swiglu, add, off, launches; };
static const int T = 8192, V = 128256;
static const Shape kStep[] = {
    {"fwd qkv", T, 3072, 2048, 0, 0, 0, 0, 0, 0, 0, 32},       {"fwd o", T, 2048, 2048, 0, 0, 0, 0, 0, 1, 0, 32},
    {"fwd gateup", T, 16384, 2048, 0, 0, 0, 0, 1, 0, 0, 32},   {"fwd down", T, 2048, 8192, 0, 0, 0, 0, 0, 1, 0, 32},
    {"dgrad qkv", T, 2048, 3072, 0, 1, 0, 0, 0, 0, 0, 16},     {"dgrad o", T, 2048, 2048, 0, 1, 0, 0, 0, 0, 0, 16},
    {"dgrad gateup", T, 2048, 16384, 0, 1, 0, 0, 0, 0, 0, 16}, {"dgrad down", T, 8192, 2048, 0, 1, 0, 0, 0, 0, 0, 16},
    {"wgrad qkv", 3072, 2048, T, 1, 1, 1, 0, 0, 0, 8, 16},     {"wgrad o", 2048, 2048, T, 1, 1, 1, 0, 0, 0, 8, 16},
    {"wgrad gateup", 16384, 2048, T, 1, 1, 1, 0, 0, 0, 8, 16}, {"wgrad down", 2048, 8192, T, 1, 1, 1, 0, 0, 0, 8, 16},
    {"lm logits", 4096, V, 2048, 0, 0, 0, 0, 0, 0, 0, 2},      {"lm dh", 4096, 2048, V, 0, 1, 0, 0, 0, 0, 0, 2},
    {"lm dW", V, 2048, 4096, 1, 1, 1, 1, 0, 0, 0, 2},
};

// Step 0 of the epilogue work: t(K) / rounds = slope * (K / 64) + intercept, ours (static) against cuBLAS.
static void fit_shapes(cublasHandle_t h) {
  printf("== fit: time per round of tiles = slope x K blocks of 64 + intercept (static scheduling, L2 flushed) ==\n");
  const int Ks[4] = {1024, 2048, 4096, 8192};
  for (const Shape& sh : kStep) {
    const long tiles = (long)((sh.M + 127) / 128) * ((sh.N + 255) / 256);
    const double rounds = (double)((tiles + num_sms - 1) / num_sms);
    double x[4], y[2][4];
    for (int i = 0; i < 4; ++i) {
      PerfResult r = perf_case(h, sh.name, sh.M, sh.N, Ks[i], sh.a_mn, sh.b_mn, 10, sh.f32, sh.acc, sh.swiglu, sh.add,
                               sh.off, 5);
      x[i] = Ks[i] / 64.0;
      y[0][i] = r.mean[0] * 1e3 / rounds;
      y[1][i] = r.mean[2] * 1e3 / rounds;
    }
    double fit[2][2];
    for (int m = 0; m < 2; ++m) {
      double sx = 0, sy = 0, sxx = 0, sxy = 0;
      for (int i = 0; i < 4; ++i) { sx += x[i]; sy += y[m][i]; sxx += x[i] * x[i]; sxy += x[i] * y[m][i]; }
      fit[m][0] = (4 * sxy - sx * sy) / (4 * sxx - sx * sx);
      fit[m][1] = (sy - fit[m][0] * sx) / 4;
    }
    printf("FIT %-14s M=%6d N=%6d rounds=%3.0f : ours %.3f us/kblock + %.2f us/round   cuBLAS %.3f us/kblock + %.2f us/round\n",
           sh.name, sh.M, sh.N, rounds, fit[0][0], fit[0][1], fit[1][0], fit[1][1]);
  }
}

int main(int argc, char** argv) {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  num_sms = prop.multiProcessorCount;
  printf("device %s, %d SMs, cc %d.%d\n", prop.name, num_sms, prop.major, prop.minor);
  if (argc > 1) cl_mask = atoi(argv[1]);
  bool do_perf = argc < 3 || atoi(argv[2]) != 0;
  bool do_num = argc < 4 || atoi(argv[3]) != 0;
  bool do_fit = argc > 4 && atoi(argv[4]) != 0;
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
    perf_case(h, "fwd qkv", T, 6144, 4096, 0, 0, 10);
    perf_case(h, "fwd o", T, 4096, 4096, 0, 0, 10);
    perf_case(h, "fwd gateup", T, 28672, 4096, 0, 0, 10);
    perf_case(h, "fwd down", T, 4096, 14336, 0, 0, 10);
    perf_case(h, "dgrad gateup", T, 4096, 28672, 0, 1, 10);
    perf_case(h, "dgrad down", T, 14336, 4096, 0, 1, 10);
    perf_case(h, "wgrad gateup", 28672, 4096, T, 1, 1, 10);
    perf_case(h, "wgrad down", 4096, 14336, T, 1, 1, 10);
    perf_case(h, "square 8k", 8192, 8192, 8192, 0, 0, 10);
    printf("== perf (T=8192 tokens, Llama-3.2-1B, the GEMMs of one bench.py step) ==\n");
    double step_ms[3] = {0, 0, 0};
    for (const Shape& sh : kStep) {
      PerfResult r = perf_case(h, sh.name, sh.M, sh.N, sh.K, sh.a_mn, sh.b_mn, 10, sh.f32, sh.acc, sh.swiglu, sh.add,
                               sh.off);
      for (int m = 0; m < 3; ++m) step_ms[m] += (double)r.mean[m] * sh.launches;
    }
    printf("GEMM time of one step (mean x launches, L2 flushed): static %.1f ms  dynamic %.1f ms  cuBLAS %.1f ms\n",
           step_ms[0], step_ms[1], step_ms[2]);
  }
  if (do_fit) {
    cublasHandle_t h;
    cublasCreate(&h);
    fit_shapes(h);
  }
  return ok ? 0 : 1;
}
