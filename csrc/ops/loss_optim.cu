// Cross-entropy (in-place gradient), fused AdamW on flat shards, squared-norm reduction, unscale/found_inf.
//
// * cross_entropy_fwd_bwd: one CTA per row of bf16 logits [n, V]; pass 1 = online max/sum (fp32), pass 2 (L2 hit)
//   overwrites the logits with d(loss)/d(logits) so the [n, V] tensor is never duplicated.  Together with the
//   chunked lm_head GEMM in Python this is the fused-linear-cross-entropy of reference ops/liger.py:72-76.
// * adamw_flat: one pass over the local fp32 master shard: reads grad (bf16 or fp32), m, v, p; applies the
//   device-resident scale (clip coefficient x 1/loss_scale, no host sync) and the found_inf skip; writes p, m, v
//   and the bf16 compute copy that the next all-gather sends.  Replaces torch fused Adam / torch_xla syncfree
//   optimizers (reference utils/patch.py:55-58).
#include "../common/ptx.cuh"
#include "ops.h"

namespace tb {

constexpr int kCEThreads = 1024;

TB_DEVICE void unpack8f(const uint4& u, float (&f)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}

// loss_rows[row] = lse - logit[label] (0 for ignored rows); logits <- (softmax - onehot) * grad_scale (0 if ignored)
// grad_scale = *scale_ptr if scale_ptr else scale_val   (typically 1 / number_of_valid_tokens)
__global__ void __launch_bounds__(kCEThreads)
cross_entropy_kernel(__nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                     float* __restrict__ loss_rows, float* __restrict__ lse_rows, int V, long long ld,
                     int ignore_index, const float* __restrict__ scale_ptr, float scale_val, int write_grad) {
  __shared__ float red_m[32], red_s[32];
  __shared__ float s_max, s_sum;
  const long long row = blockIdx.x;
  __nv_bfloat16* lr = logits + row * ld;
  const long long label = labels[row];
  const bool ignored = label == ignore_index;
  const int nvec = V >> 3;
  const float kLog2e = 1.4426950408889634f;
  // pass 1: online softmax statistics
  float m = -INFINITY, s = 0.f;
  for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
    float f[8];
    unpack8f(reinterpret_cast<const uint4*>(lr)[v], f);
    float lm = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) lm = fmaxf(lm, f[j]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += fast_exp2((f[j] - nm) * kLog2e);
    s = s * fast_exp2((m - nm) * kLog2e) + acc;
    m = nm;
  }
  for (int i = nvec * 8 + threadIdx.x; i < V; i += kCEThreads) {  // tail (V % 8 != 0)
    const float f = __bfloat162float(lr[i]);
    const float nm = fmaxf(m, f);
    s = s * fast_exp2((m - nm) * kLog2e) + fast_exp2((f - nm) * kLog2e);
    m = nm;
  }
  // block combine
  {
    float wm = warp_reduce_max(m);
    float ws = warp_reduce_sum(m == -INFINITY ? 0.f : s * fast_exp2((m - wm) * kLog2e));
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { red_m[w] = wm; red_s[w] = ws; }
    __syncthreads();
    if (w == 0) {
      float bm = red_m[l], bs = red_s[l];
      float gm = warp_reduce_max(bm);
      float gs = warp_reduce_sum(bm == -INFINITY ? 0.f : bs * fast_exp2((bm - gm) * kLog2e));
      if (l == 0) { s_max = gm; s_sum = gs; }
    }
    __syncthreads();
  }
  const float gmax = s_max, gsum = s_sum;
  const float lse = gmax + logf(gsum);
  if (threadIdx.x == 0) {
    float lab_logit = ignored ? 0.f : __bfloat162float(lr[label]);
    loss_rows[row] = ignored ? 0.f : (lse - lab_logit);
    if (lse_rows) lse_rows[row] = lse;
  }
  if (!write_grad) return;
  __syncthreads();  // label logit is read before anyone overwrites it
  const float gscale = ignored ? 0.f : (scale_ptr ? *scale_ptr : scale_val);
  const float inv_sum = 1.f / gsum;
  for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
    float f[8];
    uint4* p = reinterpret_cast<uint4*>(lr) + v;
    unpack8f(*p, f);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float pr = fast_exp2((f[j] - gmax) * kLog2e) * inv_sum;
      if ((long long)v * 8 + j == label) pr -= 1.f;
      o[j] = pr * gscale;
    }
    uint4 u;
    u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]);
    u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
    *p = u;
  }
  for (int i = nvec * 8 + threadIdx.x; i < V; i += kCEThreads) {
    float pr = fast_exp2((__bfloat162float(lr[i]) - gmax) * kLog2e) * inv_sum;
    if (i == label) pr -= 1.f;
    lr[i] = __float2bfloat16(pr * gscale);
  }
}

cudaError_t cross_entropy_fwd_bwd(void* logits, const long long* labels, float* loss_rows, float* lse_rows, int n,
                                  int V, long long ld, int ignore_index, const float* scale_ptr, float scale_val,
                                  bool write_grad, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  if (ld % 8 != 0) return cudaErrorInvalidValue;
  cross_entropy_kernel<<<n, kCEThreads, 0, stream>>>((__nv_bfloat16*)logits, labels, loss_rows, lse_rows, V, ld,
                                                     ignore_index, scale_ptr, scale_val, write_grad ? 1 : 0);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Fused AdamW over a flat fp32 shard.
// ---------------------------------------------------------------------------------------------------
template <typename GradT>
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, const GradT* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             __nv_bfloat16* __restrict__ p_lp, long long n, float lr, float beta1, float beta2, float eps,
             float weight_decay, float bc1, float bc2_sqrt, const float* __restrict__ grad_scale,
             const float* __restrict__ found_inf) {
  if (found_inf && *found_inf != 0.f) return;  // skipped step (fp16 loss scaling)
  const float gs = grad_scale ? *grad_scale : 1.f;
  const long long nvec = n >> 2;
  const float step_size = lr / bc1;
  const float decay = 1.f - lr * weight_decay;
  const float inv_bc2 = 1.f / bc2_sqrt;
  // two independent 16-byte groups per thread per trip (more bytes in flight), streaming (evict-first) accesses:
  // every byte is touched exactly once per step
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < nvec; i0 += 2 * stride) {
    float4 pp[2], mm[2], vv[2];
    float gg[2][4];
    bool on[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const long long i = i0 + k * stride;
      on[k] = i < nvec;
      if (on[k]) {
        pp[k] = __ldcs(reinterpret_cast<const float4*>(p) + i);
        mm[k] = __ldcs(reinterpret_cast<const float4*>(m) + i);
        vv[k] = __ldcs(reinterpret_cast<const float4*>(v) + i);
        if constexpr (sizeof(GradT) == 4) {
          float4 t = __ldcs(reinterpret_cast<const float4*>(g) + i);
          gg[k][0] = t.x; gg[k][1] = t.y; gg[k][2] = t.z; gg[k][3] = t.w;
        } else {
          uint2 t = __ldcs(reinterpret_cast<const uint2*>(g) + i);
          float2 a = unpack_bf16x2(t.x), b = unpack_bf16x2(t.y);
          gg[k][0] = a.x; gg[k][1] = a.y; gg[k][2] = b.x; gg[k][3] = b.y;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!on[k]) continue;
      const long long i = i0 + k * stride;
      float pa[4] = {pp[k].x, pp[k].y, pp[k].z, pp[k].w}, ma[4] = {mm[k].x, mm[k].y, mm[k].z, mm[k].w},
            va[4] = {vv[k].x, vv[k].y, vv[k].z, vv[k].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gr = gg[k][j] * gs;
        pa[j] *= decay;
        ma[j] = beta1 * ma[j] + (1.f - beta1) * gr;
        va[j] = beta2 * va[j] + (1.f - beta2) * gr * gr;
        const float denom = sqrtf(va[j]) * inv_bc2 + eps;
        pa[j] -= step_size * ma[j] / denom;
      }
      __stcs(reinterpret_cast<float4*>(p) + i, make_float4(pa[0], pa[1], pa[2], pa[3]));
      __stcs(reinterpret_cast<float4*>(m) + i, make_float4(ma[0], ma[1], ma[2], ma[3]));
      __stcs(reinterpret_cast<float4*>(v) + i, make_float4(va[0], va[1], va[2], va[3]));
      if (p_lp) {
        uint2 o;
        o.x = pack_bf16x2(pa[0], pa[1]);
        o.y = pack_bf16x2(pa[2], pa[3]);
        reinterpret_cast<uint2*>(p_lp)[i] = o;   // default policy: the bf16 copy is re-read by the next forward
      }
    }
  }
  // scalar tail
  for (long long i = (nvec << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float gr;
    if constexpr (sizeof(GradT) == 4) gr = g[i] * gs; else gr = __bfloat162float(g[i]) * gs;
    float pa = p[i] * (1.f - lr * weight_decay);
    float ma = beta1 * m[i] + (1.f - beta1) * gr;
    float va = beta2 * v[i] + (1.f - beta2) * gr * gr;
    pa -= step_size * ma / (sqrtf(va) / bc2_sqrt + eps);
    p[i] = pa; m[i] = ma; v[i] = va;
    if (p_lp) p_lp[i] = __float2bfloat16(pa);
  }
}

cudaError_t adamw_flat(float* p, const void* g, bool grad_is_bf16, float* m, float* v, void* p_lp, long long n,
                       float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                       const float* grad_scale, const float* found_inf, int num_sms, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  long long blocks = ((n >> 2) + 255) / 256;
  if (blocks < 1) blocks = 1;
  int grid = (int)(blocks < (long long)num_sms * 16 ? blocks : (long long)num_sms * 16);
  if (grad_is_bf16)
    adamw_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(p, (const __nv_bfloat16*)g, m, v, (__nv_bfloat16*)p_lp, n,
                                                          lr, beta1, beta2, eps, weight_decay, bc1, bc2_sqrt,
                                                          grad_scale, found_inf);
  else
    adamw_kernel<float><<<grid, 256, 0, stream>>>(p, (const float*)g, m, v, (__nv_bfloat16*)p_lp, n, lr, beta1, beta2,
                                                  eps, weight_decay, bc1, bc2_sqrt, grad_scale, found_inf);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// out[0] += sum(g^2) ; out[1] = 1 if any non-finite (found_inf).  Used for grad-norm clipping and GradScaler.
// ---------------------------------------------------------------------------------------------------
template <typename GradT>
__global__ void __launch_bounds__(256)
sqnorm_kernel(const GradT* __restrict__ g, long long n, float* __restrict__ out, float pre_scale) {
  __shared__ float red[8];
  float acc = 0.f;
  bool bad = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float x;
    if constexpr (sizeof(GradT) == 4) x = g[i]; else x = __bfloat162float(g[i]);
    x *= pre_scale;
    bad |= !isfinite(x);
    acc += x * x;
  }
  acc = warp_reduce_sum(acc);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = acc;
  const int any_bad = __syncthreads_or(bad ? 1 : 0);
  if (w == 0) {
    float t = l < 8 ? red[l] : 0.f;
    t = warp_reduce_sum(t);
    if (l == 0) {
      atomicAdd(out, t);
      if (any_bad) out[1] = 1.f;
    }
  }
}

cudaError_t sqnorm_accumulate(const void* g, bool is_bf16, long long n, float* out, float pre_scale, int num_sms,
                              cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  long long blocks = (n + 256 * 8 - 1) / (256 * 8);
  int grid = (int)(blocks < (long long)num_sms * 8 ? blocks : (long long)num_sms * 8);
  if (is_bf16) sqnorm_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)g, n, out, pre_scale);
  else sqnorm_kernel<float><<<grid, 256, 0, stream>>>((const float*)g, n, out, pre_scale);
  return cudaGetLastError();
}

// Deterministic variant, still one launch: every block writes its partial sum to partial[blockIdx.x] and takes an
// integer ticket; the last block to finish adds the partials in index order to out[0] and resets the counter.  Only the
// ticket order depends on scheduling, never a value, and the grid depends on n and the SM count only, so repeated
// calls give bitwise-equal sums.  found_inf is the same idempotent flag write as in sqnorm_kernel.
template <typename GradT>
__global__ void __launch_bounds__(256)
sqnorm_ordered_kernel(const GradT* __restrict__ g, long long n, float* __restrict__ out, float pre_scale,
                      float* __restrict__ partial, unsigned int* __restrict__ counter) {
  __shared__ float red[8];
  __shared__ bool last;
  float acc = 0.f;
  bool bad = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float x;
    if constexpr (sizeof(GradT) == 4) x = g[i]; else x = __bfloat162float(g[i]);
    x *= pre_scale;
    bad |= !isfinite(x);
    acc += x * x;
  }
  acc = warp_reduce_sum(acc);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = acc;
  const int any_bad = __syncthreads_or(bad ? 1 : 0);
  if (w == 0) {
    float t = l < 8 ? red[l] : 0.f;
    t = warp_reduce_sum(t);
    if (l == 0) {
      partial[blockIdx.x] = t;
      if (any_bad) out[1] = 1.f;
      __threadfence();                                   // the partial is visible before the ticket is taken
      last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  // fixed-shape reduction over the partials: thread t sums t, t + 256, ... in order, then the block tree
  float s = 0.f;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) s += __ldcg(partial + i);
  s = warp_reduce_sum(s);
  if (l == 0) red[w] = s;
  __syncthreads();
  if (w == 0) {
    float t = l < 8 ? red[l] : 0.f;
    t = warp_reduce_sum(t);
    if (l == 0) {
      out[0] += t;
      *counter = 0u;                                     // ready for the next launch on this stream
    }
  }
}

cudaError_t sqnorm_accumulate_ordered(const void* g, bool is_bf16, long long n, float* out, float pre_scale,
                                      float* partial, unsigned int* counter, int num_sms, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  long long blocks = (n + 256 * 8 - 1) / (256 * 8);     // same grid as sqnorm_accumulate: at most 8 blocks per SM
  int grid = (int)(blocks < (long long)num_sms * 8 ? blocks : (long long)num_sms * 8);
  if (is_bf16)
    sqnorm_ordered_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)g, n, out, pre_scale, partial,
                                                                   counter);
  else
    sqnorm_ordered_kernel<float><<<grid, 256, 0, stream>>>((const float*)g, n, out, pre_scale, partial, counter);
  return cudaGetLastError();
}

// g *= *scale (in place) -- GradScaler unscale / clip for optimizers that are not ours.
template <typename GradT>
__global__ void __launch_bounds__(256) scale_kernel(GradT* __restrict__ g, long long n, const float* __restrict__ scale) {
  const float s = *scale;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    if constexpr (sizeof(GradT) == 4) g[i] *= s; else g[i] = __float2bfloat16(__bfloat162float(g[i]) * s);
  }
}

cudaError_t scale_inplace(void* g, bool is_bf16, long long n, const float* scale, int num_sms, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  long long blocks = (n + 1023) / 1024;
  int grid = (int)(blocks < (long long)num_sms * 8 ? blocks : (long long)num_sms * 8);
  if (is_bf16) scale_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((__nv_bfloat16*)g, n, scale);
  else scale_kernel<float><<<grid, 256, 0, stream>>>((float*)g, n, scale);
  return cudaGetLastError();
}

}  // namespace tb
