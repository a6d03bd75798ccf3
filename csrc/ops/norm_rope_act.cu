// Bandwidth-bound transformer ops for sm_90a: RMSNorm (+fused residual add) fwd/bwd, RoPE fwd/bwd (in place,
// strided so it runs directly on the fused-QKV GEMM output), per-head QK-RMSNorm + RoPE fwd/bwd (out of place on the
// same layout), SwiGLU fwd/bwd.
// All kernels move 16 bytes per thread per access and keep rows in registers between the reduction and the
// normalisation pass, so each tensor is read exactly once and written exactly once.
// Replaces the Triton liger kernels the reference patches in (reference torchacc/ops/liger.py:10-28,69-70).
#include "../common/ptx.cuh"
#include "ops.h"

namespace tb {

constexpr int kNormThreads = 256;
constexpr int kMaxVec = 8;  // H <= 256 * 8 * 8 = 16384

struct alignas(16) bf16x8 {
  uint4 u;
};

// 8 x 16-bit floats (bf16 or fp16, kernel template parameter) <-> 8 floats
template <bool kBf16>
TB_DEVICE void unpack8(const uint4& u, float (&f)[8]) {
  float2 a = unpack_h2<kBf16>(u.x), b = unpack_h2<kBf16>(u.y), c = unpack_h2<kBf16>(u.z), d = unpack_h2<kBf16>(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
template <bool kBf16>
TB_DEVICE uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_h2<kBf16>(f[0], f[1]); u.y = pack_h2<kBf16>(f[2], f[3]);
  u.z = pack_h2<kBf16>(f[4], f[5]); u.w = pack_h2<kBf16>(f[6], f[7]);
  return u;
}

template <int kThreads>
TB_DEVICE float block_reduce_sum(float v, float* red) {
  v = warp_reduce_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < kThreads / 32) ? red[l] : 0.f;
  t = warp_reduce_sum(t);
  return t;
}

// ---------------------------------------------------------------------------------------------------
// RMSNorm forward.  y = (x [+ res]) * rstd * w ;  optionally writes h = x + res (the new residual stream).
// ---------------------------------------------------------------------------------------------------
template <int kVpt, bool kBf16>
__global__ void __launch_bounds__(kNormThreads)
rmsnorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                   const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ y,
                   __nv_bfloat16* __restrict__ h_out, float* __restrict__ rstd_out, int rows, int H, float eps) {
  __shared__ float red[32];
  const int nvec = H >> 3;
  float wv[kVpt][8];
#pragma unroll
  for (int i = 0; i < kVpt; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(w) + v), wv[i]);
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * H);
    const uint4* rr = res ? reinterpret_cast<const uint4*>(res + (size_t)row * H) : nullptr;
    float xv[kVpt][8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        unpack8<kBf16>(xr[v], xv[i]);
        if (rr) {
          float rv[8];
          unpack8<kBf16>(rr[v], rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) xv[i][j] += rv[j];
          uint4 hp = pack8<kBf16>(xv[i]);
          if (h_out) reinterpret_cast<uint4*>(h_out + (size_t)row * H)[v] = hp;
          unpack8<kBf16>(hp, xv[i]);  // normalise exactly what the residual stream stores (bf16-rounded)
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += xv[i][j] * xv[i][j];
      }
    }
    ss = block_reduce_sum<kNormThreads>(ss, red);
    const float rstd = rsqrtf(ss / (float)H + eps);
    if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = xv[i][j] * rstd * wv[i][j];
        reinterpret_cast<uint4*>(y + (size_t)row * H)[v] = pack8<kBf16>(o);
      }
    }
  }
}

// RMSNorm backward.  dx = rstd * (dy*w - xhat * mean(dy*w*xhat)) [+ dres];  dw partial sums per CTA are written to
// row blockIdx.x of dw_partial[gridDim.x, H] (fp32, no atomics; the caller sums the rows).
// The next row's x / dy / dres are prefetched as raw 16-byte vectors before the current row's block reduction, so two
// rows of loads are in flight per CTA and the reduction latency is hidden.
template <int kVpt, int kThreads, bool kBf16>
__global__ void __launch_bounds__(kThreads, (kVpt == 1) ? (1024 / kThreads) : 1)
rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                   const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd,
                   const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx,
                   float* __restrict__ dw_partial, int rows, int H) {
  __shared__ float red[32];
  const int nvec = H >> 3;
  float wv[kVpt][8], dwv[kVpt][8];
#pragma unroll
  for (int i = 0; i < kVpt; ++i) {
    const int v = threadIdx.x + i * kThreads;
    if (v < nvec) unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(w) + v), wv[i]);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwv[i][j] = 0.f;
  }
  uint4 xn[kVpt], gn[kVpt], rn[kVpt];
  float rs_n = 0.f;
  auto prefetch = [&](int row) {
    if (row < rows) {
      rs_n = rstd[row];
#pragma unroll
      for (int i = 0; i < kVpt; ++i) {
        const int v = threadIdx.x + i * kThreads;
        if (v < nvec) {
          xn[i] = reinterpret_cast<const uint4*>(x + (size_t)row * H)[v];
          gn[i] = reinterpret_cast<const uint4*>(dy + (size_t)row * H)[v];
          if (dres) rn[i] = reinterpret_cast<const uint4*>(dres + (size_t)row * H)[v];
        }
      }
    }
  };
  prefetch(blockIdx.x);
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    uint4 xc[kVpt], gc[kVpt], rc[kVpt];
    const float rs = rs_n;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) { xc[i] = xn[i]; gc[i] = gn[i]; rc[i] = rn[i]; }
    prefetch(row + gridDim.x);
    float xh[kVpt][8], gw[kVpt][8];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) {
      const int v = threadIdx.x + i * kThreads;
      if (v < nvec) {
        float g[8];
        unpack8<kBf16>(xc[i], xh[i]);
        unpack8<kBf16>(gc[i], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] *= rs;
          dwv[i][j] += g[j] * xh[i][j];
          gw[i][j] = g[j] * wv[i][j];
          dot += gw[i][j] * xh[i][j];
        }
      }
    }
    dot = block_reduce_sum<kThreads>(dot, red) / (float)H;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) {
      const int v = threadIdx.x + i * kThreads;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (gw[i][j] - xh[i][j] * dot);
        if (dres) {
          float r[8];
          unpack8<kBf16>(rc[i], r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        __stcs(reinterpret_cast<uint4*>(dx + (size_t)row * H) + v, pack8<kBf16>(o));
      }
    }
  }
  if (dw_partial) {
    float* dst = dw_partial + (size_t)blockIdx.x * H;
#pragma unroll
    for (int i = 0; i < kVpt; ++i) {
      const int v = threadIdx.x + i * kThreads;
      if (v < nvec) {
        reinterpret_cast<float4*>(dst + v * 8)[0] = make_float4(dwv[i][0], dwv[i][1], dwv[i][2], dwv[i][3]);
        reinterpret_cast<float4*>(dst + v * 8)[1] = make_float4(dwv[i][4], dwv[i][5], dwv[i][6], dwv[i][7]);
      }
    }
  }
}

cudaError_t rmsnorm_fwd(const void* x, const void* res, const void* w, void* y, void* h_out, float* rstd, int rows,
                        int H, float eps, int num_sms, bool is_bf16, cudaStream_t stream) {
  if (rows == 0) return cudaSuccess;
  if (H % 8 != 0 || H > kNormThreads * 8 * kMaxVec) return cudaErrorInvalidValue;
  int grid = rows < num_sms * 8 ? rows : num_sms * 8;
  const int vpt = (H / 8 + kNormThreads - 1) / kNormThreads;
#define TB_LAUNCH2(V, BF)                                                                                          \
  rmsnorm_fwd_kernel<V, BF><<<grid, kNormThreads, 0, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)res, \
                                                               (const __nv_bfloat16*)w, (__nv_bfloat16*)y,         \
                                                               (__nv_bfloat16*)h_out, rstd, rows, H, eps)
#define TB_LAUNCH(V) do { if (is_bf16) TB_LAUNCH2(V, true); else TB_LAUNCH2(V, false); } while (0)
  if (vpt <= 1) TB_LAUNCH(1); else if (vpt <= 2) TB_LAUNCH(2); else if (vpt <= 4) TB_LAUNCH(4); else TB_LAUNCH(8);
#undef TB_LAUNCH
#undef TB_LAUNCH2
  return cudaGetLastError();
}

cudaError_t rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                        float* dw, int dw_rows, int rows, int H, int num_sms, bool is_bf16, cudaStream_t stream) {
  if (rows == 0) return cudaSuccess;
  if (H % 8 != 0 || H > kNormThreads * 8 * kMaxVec) return cudaErrorInvalidValue;
  // dw is a [dw_rows, H] fp32 partial-sum buffer: exactly dw_rows CTAs run and each writes its own row
  int grid = dw_rows;
  if (grid < 1 || grid > rows || dw == nullptr) return cudaErrorInvalidValue;
  (void)num_sms;
  const int nvec = H / 8;
  // wide rows use 512-thread CTAs so a thread keeps at most a few 16-byte vectors (x, dy, dres; current + prefetched)
  const bool wide = nvec >= 512;
  const int threads = wide ? 512 : 256;
  const int vpt = (nvec + threads - 1) / threads;
#define TB_LAUNCH2(V, T, BF)                                                                                     \
  rmsnorm_bwd_kernel<V, T, BF><<<grid, T, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,          \
                                                        (const __nv_bfloat16*)w, rstd, (const __nv_bfloat16*)dres, \
                                                        (__nv_bfloat16*)dx, dw, rows, H)
#define TB_LAUNCH(V, T) do { if (is_bf16) TB_LAUNCH2(V, T, true); else TB_LAUNCH2(V, T, false); } while (0)
  if (wide) {
    if (vpt <= 1) TB_LAUNCH(1, 512); else if (vpt <= 2) TB_LAUNCH(2, 512); else TB_LAUNCH(4, 512);
  } else {
    if (vpt <= 1) TB_LAUNCH(1, 256); else TB_LAUNCH(2, 256);
  }
#undef TB_LAUNCH
#undef TB_LAUNCH2
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// RoPE (rotate-half convention, HF Llama): in place on x[T, nheads, D] with token stride `ts` elements.
//   out[:D/2] = x1*cos - x2*sin ; out[D/2:] = x2*cos + x1*sin        (backward: sin -> -sin)
// cos/sin tables are fp32 [max_pos, D/2]; position of token t is positions[t] or (t % seq_len).
// ---------------------------------------------------------------------------------------------------
template <bool kBf16>
__global__ void __launch_bounds__(256)
rope_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
            const int* __restrict__ positions, long long T, int nheads, int D, long long ts, int seq_len,
            float sin_sign) {
  const int half = D >> 1;
  const int vec_per_head = half >> 3;  // 8 elements per thread from each half
  const long long total = T * nheads * vec_per_head;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vec_per_head);
    const long long th = i / vec_per_head;
    const int hd = (int)(th % nheads);
    const long long t = th / nheads;
    const int pos = positions ? positions[t] : (int)(t % seq_len);
    __nv_bfloat16* base = x + t * ts + (long long)hd * D + v * 8;
    uint4 u1 = *reinterpret_cast<uint4*>(base);
    uint4 u2 = *reinterpret_cast<uint4*>(base + half);
    float a[8], b[8], c[8], s[8];
    unpack8<kBf16>(u1, a);
    unpack8<kBf16>(u2, b);
    const float4* cp = reinterpret_cast<const float4*>(cos_t + (size_t)pos * half + v * 8);
    const float4* sp = reinterpret_cast<const float4*>(sin_t + (size_t)pos * half + v * 8);
    float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
    c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
    s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sn = s[j] * sin_sign;
      o1[j] = a[j] * c[j] - b[j] * sn;
      o2[j] = b[j] * c[j] + a[j] * sn;
    }
    *reinterpret_cast<uint4*>(base) = pack8<kBf16>(o1);
    *reinterpret_cast<uint4*>(base + half) = pack8<kBf16>(o2);
  }
}

cudaError_t rope_inplace(void* x, const float* cos_t, const float* sin_t, const int* positions, long long T,
                         int nheads, int D, long long token_stride, int seq_len, bool backward, int num_sms,
                         bool is_bf16, cudaStream_t stream) {
  if (T == 0 || nheads == 0) return cudaSuccess;
  if (D % 16 != 0 || token_stride % 8 != 0) return cudaErrorInvalidValue;
  long long total = T * nheads * (D / 16);
  long long blocks = (total + 255) / 256;
  int grid = (int)(blocks < (long long)num_sms * 16 ? blocks : (long long)num_sms * 16);
  if (is_bf16)
    rope_kernel<true><<<grid, 256, 0, stream>>>((__nv_bfloat16*)x, cos_t, sin_t, positions, T, nheads, D, token_stride,
                                                 seq_len, backward ? -1.f : 1.f);
  else
    rope_kernel<false><<<grid, 256, 0, stream>>>((__nv_bfloat16*)x, cos_t, sin_t, positions, T, nheads, D,
                                                  token_stride, seq_len, backward ? -1.f : 1.f);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Per-head QK-RMSNorm + RoPE (Qwen3 q_norm / k_norm), out of place on the packed QKV layout of rope_kernel:
//   z = x * rstd * w  (rstd = rsqrt(mean(x^2) + eps), w = q_weight or k_weight),  out = rope(z)
// all in fp32 with one rounding at the end; V head rows are copied.  Backward, per row:
//   u = rope^-1(g),  xhat = x * rstd,  dx = rstd * (u w - xhat * mean(u w xhat)),  dw += u * xhat.
// A group of kQkGroup(D) lanes owns one head row: lane j holds elements [8j, 8j+8) of each half, which is exactly
// RoPE's pairing, so the sum of squares is a shuffle reduction inside the group and the row never leaves registers.
// Groups are a power of two wide (lanes past D/16 hold zeros); every lane of a warp runs every trip of the row loop so
// the shuffles see full warps.  rstd is [T, Hq + Hk] fp32; the weight gradient is written as per-CTA fp32 partials
// [gridDim.x, 2, D] (q then k), reduced in a fixed order inside the CTA: no atomics, bitwise reproducible.
// ---------------------------------------------------------------------------------------------------
constexpr int kQkThreads = 256;

__host__ __device__ __forceinline__ int qk_group(int D) {
  const int g = D >> 4;
  return g <= 1 ? 1 : g <= 2 ? 2 : g <= 4 ? 4 : g <= 8 ? 8 : 16;
}

TB_DEVICE void load_cs8(const float* __restrict__ t, size_t off, float (&f)[8]) {
  const float4* p = reinterpret_cast<const float4*>(t + off);
  const float4 a = __ldg(p), b = __ldg(p + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

TB_DEVICE float group_sum(float v, int G) {
  for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool kBf16>
__global__ void __launch_bounds__(kQkThreads)
qk_norm_rope_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                        const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw,
                        float* __restrict__ rstd_out, const float* __restrict__ cos_t,
                        const float* __restrict__ sin_t, const int* __restrict__ positions, long long T, int hq,
                        int hk, int D, long long ts, int seq_len, float eps) {
  const int G = qk_group(D), half = D >> 1, lane = threadIdx.x & 31, j = lane & (G - 1);
  const int heads = hq + 2 * hk, hqk = hq + hk;
  const bool has_cols = j * 16 < D;
  const long long rows = T * heads;
  const int rows_per_warp = 32 / G;
  const long long warp0 = (blockIdx.x * (long long)kQkThreads + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * kQkThreads) >> 5;
  for (long long wr = warp0 * rows_per_warp; wr < rows; wr += nwarps * rows_per_warp) {
    const long long row = wr + lane / G;
    const bool live = row < rows && has_cols;
    const long long t = row / heads;
    const int hd = (int)(row - t * heads);
    const long long off = t * ts + (long long)hd * D + j * 8;
    uint4 u1 = make_uint4(0, 0, 0, 0), u2 = u1;
    if (live) {
      u1 = __ldcs(reinterpret_cast<const uint4*>(x + off));
      u2 = __ldcs(reinterpret_cast<const uint4*>(x + off + half));
    }
    float a[8], b[8];
    unpack8<kBf16>(u1, a);
    unpack8<kBf16>(u2, b);
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) ss += a[e] * a[e] + b[e] * b[e];
    ss = group_sum(ss, G);
    if (!live) continue;
    if (hd >= hqk) {   // V head: copied unchanged
      __stcs(reinterpret_cast<uint4*>(out + off), u1);
      __stcs(reinterpret_cast<uint4*>(out + off + half), u2);
      continue;
    }
    const float rstd = rsqrtf(ss / (float)D + eps);
    if (j == 0) rstd_out[t * hqk + hd] = rstd;
    const __nv_bfloat16* w = hd < hq ? qw : kw;
    float wa[8], wb[8], c[8], s[8];
    unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(w + j * 8)), wa);
    unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(w + half + j * 8)), wb);
    const int pos = positions ? positions[t] : (int)(t % seq_len);
    load_cs8(cos_t, (size_t)pos * half + j * 8, c);
    load_cs8(sin_t, (size_t)pos * half + j * 8, s);
    float o1[8], o2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float za = a[e] * rstd * wa[e], zb = b[e] * rstd * wb[e];
      o1[e] = za * c[e] - zb * s[e];
      o2[e] = zb * c[e] + za * s[e];
    }
    __stcs(reinterpret_cast<uint4*>(out + off), pack8<kBf16>(o1));
    __stcs(reinterpret_cast<uint4*>(out + off + half), pack8<kBf16>(o2));
  }
}

// (two CTAs per SM: the 32 fp32 weight-gradient accumulators per thread must fit in 128 registers)
template <bool kBf16>
__global__ void __launch_bounds__(kQkThreads, 2)
qk_norm_rope_bwd_kernel(const __nv_bfloat16* __restrict__ g_, const __nv_bfloat16* __restrict__ x,
                        __nv_bfloat16* __restrict__ dx, const __nv_bfloat16* __restrict__ qw,
                        const __nv_bfloat16* __restrict__ kw, const float* __restrict__ rstd_in,
                        float* __restrict__ dw_partial, const float* __restrict__ cos_t,
                        const float* __restrict__ sin_t, const int* __restrict__ positions, long long T, int hq,
                        int hk, int D, long long ts, int seq_len) {
  // every thread's 2 x 16 weight-gradient columns, then summed over the CTA's groups in a fixed order
  __shared__ float red[kQkThreads][2][16];
  const int G = qk_group(D), half = D >> 1, lane = threadIdx.x & 31, j = lane & (G - 1);
  const int heads = hq + 2 * hk, hqk = hq + hk;
  const bool has_cols = j * 16 < D;
  const long long rows = T * heads;
  const int rows_per_warp = 32 / G;
  const long long warp0 = (blockIdx.x * (long long)kQkThreads + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * kQkThreads) >> 5;
  float dq[16], dk[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) dq[e] = dk[e] = 0.f;
  for (long long wr = warp0 * rows_per_warp; wr < rows; wr += nwarps * rows_per_warp) {
    const long long row = wr + lane / G;
    const bool live = row < rows && has_cols;
    const long long t = row / heads;
    const int hd = (int)(row - t * heads);
    const long long off = t * ts + (long long)hd * D + j * 8;
    const bool norm_row = live && hd < hqk;
    const bool is_q = hd < hq;
    uint4 g1 = make_uint4(0, 0, 0, 0), g2 = g1, x1 = g1, x2 = g1, w1 = g1, w2 = g1;
    float rstd = 0.f, c[8], s[8];
    if (live) {
      g1 = __ldcs(reinterpret_cast<const uint4*>(g_ + off));
      g2 = __ldcs(reinterpret_cast<const uint4*>(g_ + off + half));
    }
    if (norm_row) {
      x1 = __ldcs(reinterpret_cast<const uint4*>(x + off));
      x2 = __ldcs(reinterpret_cast<const uint4*>(x + off + half));
      const __nv_bfloat16* w = is_q ? qw : kw;
      w1 = __ldg(reinterpret_cast<const uint4*>(w + j * 8));
      w2 = __ldg(reinterpret_cast<const uint4*>(w + half + j * 8));
      rstd = rstd_in[t * hqk + hd];
      const int pos = positions ? positions[t] : (int)(t % seq_len);
      load_cs8(cos_t, (size_t)pos * half + j * 8, c);
      load_cs8(sin_t, (size_t)pos * half + j * 8, s);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) c[e] = s[e] = 0.f;
    }
    float ga[8], gb[8], xa[8], xb[8], wa[8], wb[8];
    unpack8<kBf16>(g1, ga);
    unpack8<kBf16>(g2, gb);
    unpack8<kBf16>(x1, xa);
    unpack8<kBf16>(x2, xb);
    unpack8<kBf16>(w1, wa);
    unpack8<kBf16>(w2, wb);
    float dot = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float ua = ga[e] * c[e] + gb[e] * s[e], ub = gb[e] * c[e] - ga[e] * s[e];   // rope^-1: sin -> -sin
      xa[e] *= rstd;
      xb[e] *= rstd;
      ga[e] = ua;  // u, kept for dw
      gb[e] = ub;
      dot += ua * wa[e] * xa[e] + ub * wb[e] * xb[e];
    }
    dot = group_sum(dot, G) / (float)D;
    if (!live) continue;
    if (!norm_row) {   // V head: the gradient passes through
      __stcs(reinterpret_cast<uint4*>(dx + off), g1);
      __stcs(reinterpret_cast<uint4*>(dx + off + half), g2);
      continue;
    }
    float o1[8], o2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      o1[e] = rstd * (ga[e] * wa[e] - xa[e] * dot);
      o2[e] = rstd * (gb[e] * wb[e] - xb[e] * dot);
      if (is_q) {
        dq[e] += ga[e] * xa[e];
        dq[8 + e] += gb[e] * xb[e];
      } else {
        dk[e] += ga[e] * xa[e];
        dk[8 + e] += gb[e] * xb[e];
      }
    }
    __stcs(reinterpret_cast<uint4*>(dx + off), pack8<kBf16>(o1));
    __stcs(reinterpret_cast<uint4*>(dx + off + half), pack8<kBf16>(o2));
  }
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    red[threadIdx.x][0][e] = dq[e];
    red[threadIdx.x][1][e] = dk[e];
  }
  __syncthreads();
  // column c of weight k (0 = q, 1 = k): element c of the row lives in lane j = (c mod half) / 8 of every group, slot
  // (c mod 8) + 8 * (c >= half); the groups are summed in thread order
  for (int i = threadIdx.x; i < 2 * D; i += kQkThreads) {
    const int which = i >= D, col = i - which * D;
    const int hi = col >= half, cj = (col - hi * half) >> 3, slot = (col & 7) + 8 * hi;
    float acc = 0.f;
    for (int th = cj; th < kQkThreads; th += G) acc += red[th][which][slot];
    dw_partial[(size_t)blockIdx.x * 2 * D + i] = acc;
  }
}

static int qk_fwd_grid(long long rows, int D, int num_sms) {
  const long long rows_per_cta = kQkThreads / qk_group(D);
  const long long blocks = (rows + rows_per_cta - 1) / rows_per_cta;
  return (int)(blocks < (long long)num_sms * 8 ? blocks : (long long)num_sms * 8);
}

cudaError_t qk_norm_rope_fwd(const void* x, void* out, const void* q_weight, const void* k_weight, float* rstd,
                             const float* cos_t, const float* sin_t, const int* positions, long long T, int hq, int hk,
                             int D, long long token_stride, int seq_len, float eps, int num_sms, bool is_bf16,
                             cudaStream_t stream) {
  if (T == 0) return cudaSuccess;
  if (D % 16 != 0 || D > 256 || token_stride % 8 != 0 || hq < 0 || hk < 0) return cudaErrorInvalidValue;
  const long long rows = T * (hq + 2 * hk);
  if (rows == 0) return cudaSuccess;
  const int grid = qk_fwd_grid(rows, D, num_sms);
#define TB_ARGS                                                                                                      \
  (const __nv_bfloat16*)x, (__nv_bfloat16*)out, (const __nv_bfloat16*)q_weight, (const __nv_bfloat16*)k_weight, rstd, \
      cos_t, sin_t, positions, T, hq, hk, D, token_stride, seq_len, eps
  if (is_bf16)
    qk_norm_rope_fwd_kernel<true><<<grid, kQkThreads, 0, stream>>>(TB_ARGS);
  else
    qk_norm_rope_fwd_kernel<false><<<grid, kQkThreads, 0, stream>>>(TB_ARGS);
#undef TB_ARGS
  return cudaGetLastError();
}

cudaError_t qk_norm_rope_bwd(const void* g, const void* x, void* dx, const void* q_weight, const void* k_weight,
                             const float* rstd, float* dw_partial, int dw_rows, const float* cos_t, const float* sin_t,
                             const int* positions, long long T, int hq, int hk, int D, long long token_stride,
                             int seq_len, int num_sms, bool is_bf16, cudaStream_t stream) {
  (void)num_sms;
  if (D % 16 != 0 || D > 256 || token_stride % 8 != 0 || hq < 0 || hk < 0) return cudaErrorInvalidValue;
  // dw_partial is [dw_rows, 2, D] fp32: exactly dw_rows CTAs run and each writes its own row (zeros if it has no work)
  if (dw_rows < 1 || dw_partial == nullptr) return cudaErrorInvalidValue;
#define TB_ARGS                                                                                                   \
  (const __nv_bfloat16*)g, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx, (const __nv_bfloat16*)q_weight,          \
      (const __nv_bfloat16*)k_weight, rstd, dw_partial, cos_t, sin_t, positions, T, hq, hk, D, token_stride, seq_len
  if (is_bf16)
    qk_norm_rope_bwd_kernel<true><<<dw_rows, kQkThreads, 0, stream>>>(TB_ARGS);
  else
    qk_norm_rope_bwd_kernel<false><<<dw_rows, kQkThreads, 0, stream>>>(TB_ARGS);
#undef TB_ARGS
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// SwiGLU: h = silu(g) * u.  g and u are separate row-strided matrices [T, F] (for the fused gate|up projection
// u = g + F and both strides are 2F); h is [T, F] contiguous.  sigmoid is fast_sigmoid (common/ptx.cuh): ex2 + rcp,
// no IEEE divide and its fix-up code.
// ---------------------------------------------------------------------------------------------------
// One CTA walks whole rows (no per-element index division); two independent 16-byte vector pairs per thread and
// iteration keep 4 loads in flight per thread.
template <bool kBf16>
__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ g_, const __nv_bfloat16* __restrict__ u_,
                  __nv_bfloat16* __restrict__ h, long long T, int F, long long ldg, long long ldu) {
  const int vpr = F >> 3;
  for (long long t = blockIdx.x; t < T; t += gridDim.x) {
    const uint4* gp = reinterpret_cast<const uint4*>(g_ + t * ldg);
    const uint4* up = reinterpret_cast<const uint4*>(u_ + t * ldu);
    uint4* hp = reinterpret_cast<uint4*>(h + t * (long long)F);
    for (int v = threadIdx.x; v < vpr; v += 512) {
      const int v1 = v + 256;
      const bool has1 = v1 < vpr;
      const uint4 gr0 = __ldcs(gp + v), ur0 = __ldcs(up + v);
      uint4 gr1 = gr0, ur1 = ur0;
      if (has1) { gr1 = __ldcs(gp + v1); ur1 = __ldcs(up + v1); }
      float g[8], u[8], o[8];
      unpack8<kBf16>(gr0, g); unpack8<kBf16>(ur0, u);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j] * fast_sigmoid(g[j]) * u[j];
      hp[v] = pack8<kBf16>(o);
      if (has1) {
        unpack8<kBf16>(gr1, g); unpack8<kBf16>(ur1, u);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = g[j] * fast_sigmoid(g[j]) * u[j];
        hp[v1] = pack8<kBf16>(o);
      }
    }
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(256)
swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ g_,
                  const __nv_bfloat16* __restrict__ u_, __nv_bfloat16* __restrict__ dg_,
                  __nv_bfloat16* __restrict__ du_, long long T, int F, long long ldg, long long ldu, long long lddg,
                  long long lddu) {
  const int vpr = F >> 3;
  for (long long t = blockIdx.x; t < T; t += gridDim.x) {
    const uint4* gp = reinterpret_cast<const uint4*>(g_ + t * ldg);
    const uint4* up = reinterpret_cast<const uint4*>(u_ + t * ldu);
    const uint4* dp = reinterpret_cast<const uint4*>(dh + t * (long long)F);
    uint4* dgp = reinterpret_cast<uint4*>(dg_ + t * lddg);
    uint4* dup = reinterpret_cast<uint4*>(du_ + t * lddu);
    for (int v = threadIdx.x; v < vpr; v += 512) {
      const int v1 = v + 256;
      const bool has1 = v1 < vpr;
      const uint4 gr0 = __ldcs(gp + v), ur0 = __ldcs(up + v), dr0 = __ldcs(dp + v);
      uint4 gr1 = gr0, ur1 = ur0, dr1 = dr0;
      if (has1) { gr1 = __ldcs(gp + v1); ur1 = __ldcs(up + v1); dr1 = __ldcs(dp + v1); }
      float g[8], u[8], d[8], dg[8], du[8];
      unpack8<kBf16>(gr0, g); unpack8<kBf16>(ur0, u); unpack8<kBf16>(dr0, d);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float sg = fast_sigmoid(g[j]);
        const float silu = g[j] * sg;
        du[j] = d[j] * silu;
        dg[j] = d[j] * u[j] * (sg + silu * (1.f - sg));
      }
      dgp[v] = pack8<kBf16>(dg);
      dup[v] = pack8<kBf16>(du);
      if (has1) {
        unpack8<kBf16>(gr1, g); unpack8<kBf16>(ur1, u); unpack8<kBf16>(dr1, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float sg = fast_sigmoid(g[j]);
          const float silu = g[j] * sg;
          du[j] = d[j] * silu;
          dg[j] = d[j] * u[j] * (sg + silu * (1.f - sg));
        }
        dgp[v1] = pack8<kBf16>(dg);
        dup[v1] = pack8<kBf16>(du);
      }
    }
  }
}

cudaError_t swiglu_fwd(const void* g, const void* u, void* h, long long T, int F, long long ldg, long long ldu,
                       int num_sms, bool is_bf16, cudaStream_t stream) {
  if (T == 0) return cudaSuccess;
  if (F % 8 != 0 || ldg % 8 != 0 || ldu % 8 != 0) return cudaErrorInvalidValue;
  int grid = (int)(T < (long long)num_sms * 8 ? T : (long long)num_sms * 8);
  if (is_bf16)
    swiglu_fwd_kernel<true><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)g, (const __nv_bfloat16*)u,
                                                       (__nv_bfloat16*)h, T, F, ldg, ldu);
  else
    swiglu_fwd_kernel<false><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)g, (const __nv_bfloat16*)u,
                                                        (__nv_bfloat16*)h, T, F, ldg, ldu);
  return cudaGetLastError();
}

cudaError_t swiglu_bwd(const void* dh, const void* g, const void* u, void* dg, void* du, long long T, int F,
                       long long ldg, long long ldu, long long lddg, long long lddu, int num_sms, bool is_bf16,
                       cudaStream_t stream) {
  if (T == 0) return cudaSuccess;
  if (F % 8 != 0 || ldg % 8 != 0 || ldu % 8 != 0 || lddg % 8 != 0 || lddu % 8 != 0) return cudaErrorInvalidValue;
  int grid = (int)(T < (long long)num_sms * 8 ? T : (long long)num_sms * 8);
  if (is_bf16)
    swiglu_bwd_kernel<true><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)dh, (const __nv_bfloat16*)g,
                                                       (const __nv_bfloat16*)u, (__nv_bfloat16*)dg,
                                                       (__nv_bfloat16*)du, T, F, ldg, ldu, lddg, lddu);
  else
    swiglu_bwd_kernel<false><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)dh, (const __nv_bfloat16*)g,
                                                        (const __nv_bfloat16*)u, (__nv_bfloat16*)dg,
                                                        (__nv_bfloat16*)du, T, F, ldg, ldu, lddg, lddu);
  return cudaGetLastError();
}

}  // namespace tb
