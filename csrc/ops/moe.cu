// Mixture-of-experts routing kernels for sm_90a: router (softmax -> top-k -> optional renormalisation) forward and
// backward, the expert index build, the permutation of tokens into the expert-sorted, 128-row-padded layout the grouped
// GEMMs read (gemm/gemm_bf16.cu, GroupArgs), its transpose, and the weighted combine.
//
// Every kernel is deterministic by construction: no float atomics, every sum runs in a fixed order.  The index build
// is one CTA, so the stable order inside an expert (ascending flattened (token, slot) index, equal to
// torch.argsort(expert_ids.flatten(), stable=True)) never depends on scheduling.  Counts stay on the device.
#include "../common/ptx.cuh"
#include "ops.h"

namespace tb {

constexpr int kMoeMaxExperts = 256;
constexpr int kMoeMaxTopK = 8;
constexpr int kMoeTile = 128;   // kBlockM of the grouped GEMM: every expert segment is padded to a multiple of it
constexpr int kIndexThreads = 1024;
constexpr int kRowThreads = 256;

// logits dtype: 0 = fp32, 1 = bf16, 2 = fp16
template <int kDt>
TB_DEVICE float ld_logit(const void* p, long long i) {
  if constexpr (kDt == 0) return reinterpret_cast<const float*>(p)[i];
  else if constexpr (kDt == 1) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  else return __half2float(reinterpret_cast<const __half*>(p)[i]);
}
template <int kDt>
TB_DEVICE void st_logit(void* p, long long i, float v) {
  if constexpr (kDt == 0) reinterpret_cast<float*>(p)[i] = v;
  else if constexpr (kDt == 1) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16(v);
  else reinterpret_cast<__half*>(p)[i] = __float2half(v);
}

// Softmax over the E logits of one token, held by one warp: lane l owns experts l, l + 32, ... (fp32 probabilities).
template <int kDt>
TB_DEVICE void warp_softmax(const void* logits, long long t, int E, float (&p)[kMoeMaxExperts / 32]) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    const int e = lane + 32 * i;
    p[i] = e < E ? ld_logit<kDt>(logits, t * E + e) : -INFINITY;
    mx = fmaxf(mx, p[i]);
  }
  mx = warp_reduce_max(mx);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    const int e = lane + 32 * i;
    p[i] = e < E ? expf(p[i] - mx) : 0.f;
    s += p[i];
  }
  s = warp_reduce_sum(s);
  const float inv = 1.f / s;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) p[i] *= inv;
}

// probability of expert e (owned by lane e % 32) broadcast to the whole warp
TB_DEVICE float warp_prob(const float (&p)[kMoeMaxExperts / 32], int e) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i)
    if (i == e / 32) v = p[i];
  return __shfl_sync(0xffffffffu, v, e & 31);
}

template <int kDt>
__global__ void __launch_bounds__(256)
moe_router_fwd_kernel(const void* __restrict__ logits, float* __restrict__ weights, long long* __restrict__ ids, int T,
                      int E, int k, bool norm) {
  const long long t = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (t >= T) return;
  const int lane = threadIdx.x & 31;
  float p[kMoeMaxExperts / 32];
  warp_softmax<kDt>(logits, t, E, p);
  bool taken[kMoeMaxExperts / 32];
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) taken[i] = false;
  float w[kMoeMaxTopK];
  int sel[kMoeMaxTopK];
  float sum = 0.f;
  for (int j = 0; j < k; ++j) {
    // warp argmax over the experts not yet taken; ties go to the lower expert index.  NaN ranks above every number, as
    // in torch.topk: a non-finite logit turns the whole row into NaN probabilities, and the row must still pick k
    // distinct experts in [0, E) (with NaN weights) rather than the out-of-range id E that the index build drops.
    float bv = -1.f;
    int be = E;
#pragma unroll
    for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
      const int e = lane + 32 * i;
      if (e < E && !taken[i] && (p[i] > bv || (isnan(p[i]) && !isnan(bv)))) { bv = p[i]; be = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      const bool on = isnan(ov), bn = isnan(bv);
      if (ov > bv || (ov == bv && oe < be) || (on && (!bn || oe < be))) { bv = ov; be = oe; }
    }
#pragma unroll
    for (int i = 0; i < kMoeMaxExperts / 32; ++i)
      if (lane + 32 * i == be) taken[i] = true;
    w[j] = bv;
    sel[j] = be;
    sum += bv;
  }
  if (lane < k) {
    float wj = 0.f;
    int ej = 0;
    for (int j = 0; j < k; ++j)
      if (j == lane) { wj = w[j]; ej = sel[j]; }
    weights[t * k + lane] = norm ? wj / sum : wj;
    ids[t * k + lane] = ej;
  }
}

// d(weights) -> d(logits).  With renormalisation w_j = p_j / S (S = sum of the k chosen p):
//   dL/dp_j = (dw_j - sum_l dw_l w_l) / S for chosen j, 0 otherwise;   dz_m = p_m (g_m - sum_i p_i g_i).
template <int kDt>
__global__ void __launch_bounds__(256)
moe_router_bwd_kernel(const void* __restrict__ logits, const long long* __restrict__ ids,
                      const float* __restrict__ dweights, void* __restrict__ dlogits, int T, int E, int k, bool norm) {
  const long long t = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (t >= T) return;
  const int lane = threadIdx.x & 31;
  float p[kMoeMaxExperts / 32];
  warp_softmax<kDt>(logits, t, E, p);
  float S = 0.f, dot = 0.f;
  for (int j = 0; j < k; ++j) {
    const int e = (int)ids[t * k + j];
    S += warp_prob(p, e);
  }
  for (int j = 0; j < k; ++j) {
    const int e = (int)ids[t * k + j];
    dot += dweights[t * k + j] * warp_prob(p, e) / S;
  }
  float g[kMoeMaxExperts / 32];
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) g[i] = 0.f;
  float pg = 0.f;   // sum_i p_i g_i over the chosen experts
  for (int j = 0; j < k; ++j) {
    const int e = (int)ids[t * k + j];
    const float dw = dweights[t * k + j];
    const float gj = norm ? (dw - dot) / S : dw;
    pg += warp_prob(p, e) * gj;
#pragma unroll
    for (int i = 0; i < kMoeMaxExperts / 32; ++i)
      if (lane + 32 * i == e) g[i] += gj;
  }
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    const int e = lane + 32 * i;
    if (e < E) st_logit<kDt>(dlogits, t * E + e, p[i] * (g[i] - pg));
  }
}

cudaError_t moe_router_fwd(const void* logits, float* weights, long long* ids, int T, int E, int k, bool norm,
                           int dtype, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (E < 1 || E > kMoeMaxExperts || k < 1 || k > kMoeMaxTopK || k > E) return cudaErrorInvalidValue;
  const unsigned blocks = (unsigned)((T + 7) / 8);
  if (dtype == 0) moe_router_fwd_kernel<0><<<blocks, 256, 0, stream>>>(logits, weights, ids, T, E, k, norm);
  else if (dtype == 1) moe_router_fwd_kernel<1><<<blocks, 256, 0, stream>>>(logits, weights, ids, T, E, k, norm);
  else moe_router_fwd_kernel<2><<<blocks, 256, 0, stream>>>(logits, weights, ids, T, E, k, norm);
  return cudaGetLastError();
}

cudaError_t moe_router_bwd(const void* logits, const long long* ids, const float* dweights, void* dlogits, int T, int E,
                           int k, bool norm, int dtype, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (E < 1 || E > kMoeMaxExperts || k < 1 || k > kMoeMaxTopK || k > E) return cudaErrorInvalidValue;
  const unsigned blocks = (unsigned)((T + 7) / 8);
  if (dtype == 0) moe_router_bwd_kernel<0><<<blocks, 256, 0, stream>>>(logits, ids, dweights, dlogits, T, E, k, norm);
  else if (dtype == 1) moe_router_bwd_kernel<1><<<blocks, 256, 0, stream>>>(logits, ids, dweights, dlogits, T, E, k, norm);
  else moe_router_bwd_kernel<2><<<blocks, 256, 0, stream>>>(logits, ids, dweights, dlogits, T, E, k, norm);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Index build (one CTA).  Entries are processed in rounds of 1024 in flattened (token, slot) order; within a round a
// warp ranks equal experts with __match_any_sync and the 32 warps' counts are scanned per expert, so every entry's rank
// inside its expert is the number of earlier entries with the same expert.
//   pos[i]      row of entry i in the sorted buffer (offsets[e] + rank), -1 for an expert id outside [0, E)
//   row_src[r]  entry whose row r is (-1: padding row), for r < rows
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kIndexThreads)
moe_index_kernel(const long long* __restrict__ ids, int n, int E, int rows, int* __restrict__ counts,
                 int* __restrict__ offsets, int* __restrict__ tile_expert, int* __restrict__ num_m_tiles,
                 int* __restrict__ pos, int* __restrict__ row_src) {
  __shared__ int s_warp[kIndexThreads / 32][kMoeMaxExperts];
  __shared__ int s_cnt[kMoeMaxExperts];
  __shared__ int s_off[kMoeMaxExperts + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int r = tid; r < rows; r += kIndexThreads) row_src[r] = -1;
  for (int e = tid; e < E; e += kIndexThreads) s_cnt[e] = 0;
  __syncthreads();
  const unsigned lt_mask = (1u << lane) - 1u;
  for (int base = 0; base < n; base += kIndexThreads) {
    const int i = base + tid;
    const long long id = i < n ? ids[i] : -1;
    const int e = (id >= 0 && id < E) ? (int)id : -1;   // range check in 64 bits: 2^32 + 3 is not expert 3
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    for (int j = tid; j < (kIndexThreads / 32) * E; j += kIndexThreads) s_warp[j / E][j % E] = 0;
    __syncthreads();
    if (e >= 0 && (peers & lt_mask) == 0) s_warp[warp][e] = __popc(peers);
    __syncthreads();
    for (int x = tid; x < E; x += kIndexThreads) {   // exclusive scan over the warps, on top of the earlier rounds
      int run = s_cnt[x];
      for (int w = 0; w < kIndexThreads / 32; ++w) {
        const int c = s_warp[w][x];
        s_warp[w][x] = run;
        run += c;
      }
      s_cnt[x] = run;
    }
    __syncthreads();
    if (i < n) pos[i] = e >= 0 ? s_warp[warp][e] + __popc(peers & lt_mask) : -1;   // rank inside the expert
    __syncthreads();
  }
  if (tid == 0) {
    int off = 0;
    for (int x = 0; x < E; ++x) {
      s_off[x] = off;
      off += (s_cnt[x] + kMoeTile - 1) / kMoeTile * kMoeTile;
    }
    s_off[E] = off;
    *num_m_tiles = off / kMoeTile;
  }
  __syncthreads();
  for (int x = tid; x < E; x += kIndexThreads) counts[x] = s_cnt[x];
  for (int x = tid; x <= E; x += kIndexThreads) offsets[x] = s_off[x];
  const int tiles = s_off[E] / kMoeTile;
  for (int m = tid; m < tiles; m += kIndexThreads) {   // owner of tile m: the last expert starting at or before it
    const int row = m * kMoeTile;
    int lo = 0, hi = E - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_off[mid] <= row) lo = mid; else hi = mid - 1;
    }
    tile_expert[m] = lo;
  }
  for (int i = tid; i < n; i += kIndexThreads) {
    const int rank = pos[i];   // written by this same thread in the rounds above
    if (rank < 0) continue;
    const int p = s_off[(int)ids[i]] + rank;
    pos[i] = p;
    row_src[p] = i;
  }
}

cudaError_t moe_index(const long long* ids, int T, int k, int E, int rows, int* counts, int* offsets, int* tile_expert,
                      int* num_m_tiles, int* pos, int* row_src, cudaStream_t stream) {
  if (E < 1 || E > kMoeMaxExperts || k < 1 || T < 0 || rows % kMoeTile != 0) return cudaErrorInvalidValue;
  // the padded layout must fit: every expert adds at most kMoeTile - 1 padding rows
  if ((long long)rows < (long long)T * k + (long long)E * (kMoeTile - 1)) return cudaErrorInvalidValue;
  moe_index_kernel<<<1, kIndexThreads, 0, stream>>>(ids, T * k, E, rows, counts, offsets, tile_expert, num_m_tiles, pos,
                                                     row_src);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Row movers: one CTA per row (grid-strided), 16 bytes per thread per access, H % 8 == 0.
// ---------------------------------------------------------------------------------------------------
template <bool kBf16>
TB_DEVICE void unpack8f(const uint4& u, float (&f)[8]) {
  float2 a = unpack_h2<kBf16>(u.x), b = unpack_h2<kBf16>(u.y), c = unpack_h2<kBf16>(u.z), d = unpack_h2<kBf16>(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
template <bool kBf16>
TB_DEVICE uint4 pack8f(const float (&f)[8]) {
  uint4 u;
  u.x = pack_h2<kBf16>(f[0], f[1]); u.y = pack_h2<kBf16>(f[2], f[3]);
  u.z = pack_h2<kBf16>(f[4], f[5]); u.w = pack_h2<kBf16>(f[6], f[7]);
  return u;
}

// x_perm[r] = x[row_src[r] / k], zero for padding rows; rows past offsets[E] are never read and are left alone
__global__ void __launch_bounds__(kRowThreads)
moe_permute_kernel(const uint4* __restrict__ x, const int* __restrict__ row_src, const int* __restrict__ offsets,
                   uint4* __restrict__ x_perm, int k, int E, int vecs) {
  const int used = offsets[E];
  for (int r = blockIdx.x; r < used; r += gridDim.x) {
    const int s = row_src[r];
    uint4* dst = x_perm + (long long)r * vecs;
    if (s < 0) {
      for (int v = threadIdx.x; v < vecs; v += kRowThreads) dst[v] = make_uint4(0u, 0u, 0u, 0u);
    } else {
      const uint4* src = x + (long long)(s / k) * vecs;
      for (int v = threadIdx.x; v < vecs; v += kRowThreads) dst[v] = src[v];
    }
  }
}

// dx[t] = sum_j dx_perm[pos[t, j]] in fp32, j ascending
template <bool kBf16>
__global__ void __launch_bounds__(kRowThreads)
moe_unpermute_sum_kernel(const uint4* __restrict__ dx_perm, const int* __restrict__ pos, uint4* __restrict__ dx, int T,
                         int k, int vecs) {
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    for (int v = threadIdx.x; v < vecs; v += kRowThreads) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < k; ++j) {
        const int p = pos[(long long)t * k + j];
        if (p < 0) continue;
        float f[8];
        unpack8f<kBf16>(dx_perm[(long long)p * vecs + v], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
      }
      dx[(long long)t * vecs + v] = pack8f<kBf16>(acc);
    }
  }
}

// out[t] = sum_j w[t, j] y_perm[pos[t, j]] (+ residual[t]) in fp32, j ascending
template <bool kBf16>
__global__ void __launch_bounds__(kRowThreads)
moe_combine_fwd_kernel(const uint4* __restrict__ y_perm, const int* __restrict__ pos, const float* __restrict__ w,
                       const uint4* __restrict__ residual, uint4* __restrict__ out, int T, int k, int vecs) {
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    for (int v = threadIdx.x; v < vecs; v += kRowThreads) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < k; ++j) {
        const int p = pos[(long long)t * k + j];
        if (p < 0) continue;
        const float wj = w[(long long)t * k + j];
        float f[8];
        unpack8f<kBf16>(y_perm[(long long)p * vecs + v], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = fmaf(wj, f[q], acc[q]);
      }
      if (residual != nullptr) {
        float f[8];
        unpack8f<kBf16>(residual[(long long)t * vecs + v], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
      }
      out[(long long)t * vecs + v] = pack8f<kBf16>(acc);
    }
  }
}

// Per sorted row r (one CTA): dy_perm[r] = w[s] dout[t] and dw[s] = <y_perm[r], dout[t]> for s = row_src[r],
// t = s / k; padding rows are zeroed (the grouped wgrad reads them).  The dot product reduces in a fixed order.
template <bool kBf16>
__global__ void __launch_bounds__(kRowThreads)
moe_combine_bwd_kernel(const uint4* __restrict__ dout, const uint4* __restrict__ y_perm, const int* __restrict__ row_src,
                       const int* __restrict__ offsets, const float* __restrict__ w, uint4* __restrict__ dy_perm,
                       float* __restrict__ dw, int k, int E, int vecs) {
  __shared__ float red[kRowThreads / 32];
  const int used = offsets[E];
  for (int r = blockIdx.x; r < used; r += gridDim.x) {
    const int s = row_src[r];
    uint4* dst = dy_perm + (long long)r * vecs;
    if (s < 0) {
      for (int v = threadIdx.x; v < vecs; v += kRowThreads) dst[v] = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const float ws = w[s];
    const uint4* g = dout + (long long)(s / k) * vecs;
    const uint4* y = y_perm + (long long)r * vecs;
    float dot = 0.f;
    for (int v = threadIdx.x; v < vecs; v += kRowThreads) {
      float fg[8], fy[8], o[8];
      unpack8f<kBf16>(g[v], fg);
      unpack8f<kBf16>(y[v], fy);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        o[q] = ws * fg[q];
        dot = fmaf(fy[q], fg[q], dot);
      }
      dst[v] = pack8f<kBf16>(o);
    }
    dot = warp_reduce_sum(dot);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int i = 0; i < kRowThreads / 32; ++i) tot += red[i];
      dw[s] = tot;
    }
    __syncthreads();
  }
}

static unsigned row_blocks(long long rows, int num_sms) {
  long long b = (long long)num_sms * 8;
  if (b > rows) b = rows;
  return (unsigned)(b < 1 ? 1 : b);
}

cudaError_t moe_permute(const void* x, const int* row_src, const int* offsets, void* x_perm, int rows, int k, int E,
                        int H, int num_sms, cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  if (H % 8 != 0) return cudaErrorInvalidValue;
  moe_permute_kernel<<<row_blocks(rows, num_sms), kRowThreads, 0, stream>>>(
      (const uint4*)x, row_src, offsets, (uint4*)x_perm, k, E, H / 8);
  return cudaGetLastError();
}

cudaError_t moe_unpermute_sum(const void* dx_perm, const int* pos, void* dx, int T, int k, int H, int num_sms,
                              bool is_bf16, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (H % 8 != 0) return cudaErrorInvalidValue;
  auto kern = is_bf16 ? moe_unpermute_sum_kernel<true> : moe_unpermute_sum_kernel<false>;
  kern<<<row_blocks(T, num_sms), kRowThreads, 0, stream>>>((const uint4*)dx_perm, pos, (uint4*)dx, T, k, H / 8);
  return cudaGetLastError();
}

cudaError_t moe_combine_fwd(const void* y_perm, const int* pos, const float* w, const void* residual, void* out, int T,
                            int k, int H, int num_sms, bool is_bf16, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (H % 8 != 0) return cudaErrorInvalidValue;
  auto kern = is_bf16 ? moe_combine_fwd_kernel<true> : moe_combine_fwd_kernel<false>;
  kern<<<row_blocks(T, num_sms), kRowThreads, 0, stream>>>((const uint4*)y_perm, pos, w, (const uint4*)residual,
                                                            (uint4*)out, T, k, H / 8);
  return cudaGetLastError();
}

cudaError_t moe_combine_bwd(const void* dout, const void* y_perm, const int* row_src, const int* offsets, const float* w,
                            void* dy_perm, float* dw, int rows, int k, int E, int H, int num_sms, bool is_bf16,
                            cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  if (H % 8 != 0) return cudaErrorInvalidValue;
  auto kern = is_bf16 ? moe_combine_bwd_kernel<true> : moe_combine_bwd_kernel<false>;
  kern<<<row_blocks(rows, num_sms), kRowThreads, 0, stream>>>((const uint4*)dout, (const uint4*)y_perm, row_src,
                                                               offsets, w, (uint4*)dy_perm, dw, k, E, H / 8);
  return cudaGetLastError();
}

}  // namespace tb
