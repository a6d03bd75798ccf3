// FlashAttention backward on wgmma / TMA for sm_90a.
//
// One CTA per (128-key tile, kv head, batch); it loops over the q heads of the GQA group and over the 64-row query
// tiles that can see this key tile, so dK/dV are accumulated in registers with no atomics.  Two MMA warpgroups own 64
// keys each and never wait for one another.  The score tile is computed TRANSPOSED (S^T = K Q^T: accumulator rows =
// keys, columns = queries), which lets every later GEMM take its operands in place:
//   (a) S^T  = K  Q^T    A = K  (smem, K-major)          B = Q  (smem, K-major)
//   (b) dP^T = V  dO^T   A = V  (smem, K-major)          B = dO (smem, K-major)
//   in registers:  P^T = exp2(S^T*scale - LSE), dS^T = P^T o (dP^T - delta) * scale
//   (c) dV  += P^T dO    A = P^T  (registers)            B = dO (smem, MN-major)
//   (d) dK  += dS^T Q    A = dS^T (registers)            B = Q  (smem, MN-major)
//   (e) dQ   = dS K      A = dS^T (smem, read MN-major)  B = K  (smem, MN-major), over the warpgroup's 64 keys
// dQ partial tiles are reduced into the fp32 accumulator with vector red.global.add.
// Q/dO tiles stream through a 2-stage TMA ring; K/V stay resident.
//
// Reference parity: FA2 backward reached by reference torchacc/ops/flash_attn.py:56,152,206,252,301.
#include <math.h>
#include <stdio.h>

#include "../common/ptx.cuh"
#include "../common/tensormap.h"
#include "attn.h"
#include "dropout.cuh"

namespace tb {

constexpr int kTile = 128;        // keys per CTA
constexpr int kQTile = 64;        // query rows per iteration
constexpr int kBwdThreads = 384;  // producer warpgroup + 2 MMA warpgroups (64 keys each)
constexpr int kQStages = 2;

struct BwdArgs {
  const float* lse;
  const float* delta;
  float* dq_acc;
  uint16_t* dk;                // bf16 or fp16 (kernel template)
  uint16_t* dv;
  const float* alibi;          // optional ALiBi slopes [Hq] (alibi_bs == 0) or [B, Hq]
  int alibi_bs;
  const int* cu_q;
  const int* cu_k;
  int B, Sq, Sk, Hq, Hk;
  long long Tq;
  long long dk_ts, dv_ts;
  float scale_log2, scale;
  int causal, wl, wr;
  int q_bs, q_off, k_bs, k_off;   // fixed-length addressing (attn.h BlockView)
  DropoutParams drop;             // used by the kDrop instantiations only
  long long* trace;   // optional [64 iterations][16 slots] clock64 stamps of CTA (0,0,0) (debug / profiling)
};

template <int D>
struct BwdSmem {
  static constexpr int kChunks = D / 64;
  static constexpr int kKVBytes = kTile * D * 2;
  static constexpr int kQBytes = kQTile * D * 2;
  static constexpr int kK = 0;
  static constexpr int kV = kK + kKVBytes;
  static constexpr int kQ = kV + kKVBytes;
  static constexpr int kDO = kQ + kQStages * kQBytes;
  static constexpr int kDS = kDO + kQStages * kQBytes;      // dS^T [128 keys][64 queries], one 128-byte row per key
  static constexpr int kStat = kDS + kTile * kQTile * 2;    // per warpgroup: lse2[64], delta[64]
  static constexpr int kBar = kStat + 2 * 2 * kQTile * 4;
  static constexpr int kTotal = kBar + 128 + 1024;
};

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

template <int D, bool kBf16, bool kDrop>
__global__ void __launch_bounds__(kBwdThreads, 1)
flash_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                 const BwdArgs args) {
  using S = BwdSmem<D>;
  constexpr int kChunks = S::kChunks;
  constexpr int kQChunk = kQTile * 128;   // bytes of one 64-column chunk of a Q / dO stage

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();
  const int b = blockIdx.z, hk = blockIdx.y, jt = blockIdx.x;
  const int group = args.Hq / args.Hk;
  const int q_start = args.cu_q ? args.cu_q[b] : b * args.q_bs + args.q_off;
  const int q_len = args.cu_q ? (args.cu_q[b + 1] - q_start) : args.Sq;
  const int k_start = args.cu_k ? args.cu_k[b] : b * args.k_bs + args.k_off;
  const int k_len = args.cu_k ? (args.cu_k[b + 1] - k_start) : args.Sk;
  const int n0 = jt * kTile;
  if (n0 >= k_len) return;

  // query rows that can see keys [n0, n0+127]
  const int shift = k_len - q_len;
  int wr_eff = args.wr;
  if (args.causal) wr_eff = (args.wr < 0) ? 0 : min(args.wr, 0);
  const int n_last = min(n0 + kTile, k_len) - 1;
  const int i_lo = (wr_eff < 0) ? 0 : max(0, n0 - shift - wr_eff);
  const int i_hi = (args.wl < 0) ? (q_len - 1) : min(q_len - 1, n_last - shift + args.wl);
  const int it_lo = i_lo / kQTile;
  const int n_qt = (i_hi < i_lo) ? 0 : (i_hi / kQTile - it_lo + 1);
  const int n_iter = n_qt * group;

  if (n_iter == 0) {  // no query sees these keys: dK = dV = 0
    for (int r = threadIdx.x; r < min(kTile, k_len - n0); r += blockDim.x) {
      uint16_t* pk = args.dk + (long long)(k_start + n0 + r) * args.dk_ts + (long long)hk * D;
      uint16_t* pv = args.dv + (long long)(k_start + n0 + r) * args.dv_ts + (long long)hk * D;
      for (int d = 0; d < D; ++d) { pk[d] = 0; pv[d] = 0; }
    }
    return;
  }

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = base + S::kK, sV = base + S::kV, sQ = base + S::kQ, sDO = base + S::kDO, sDS = base + S::kDS;
  float* stat_all = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + S::kStat);
  const uint32_t bar = base + S::kBar;
  const uint32_t kv_full = bar;
  auto qdo_full = [&](int s) { return bar + 8u * (1 + s); };
  auto qdo_empty = [&](int s) { return bar + 8u * (1 + kQStages + s); };

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v); tma_prefetch_desc(&tmap_do);
  }
  if (warp_idx == 1 && lane == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < kQStages; ++s) { mbar_init(qdo_full(s), 1); mbar_init(qdo_empty(s), 2); }
    fence_mbar_init();
  }
  __syncthreads();

  // iteration -> (q head, q tile): heads outer, tiles inner
  auto iter_head = [&](int it) { return hk * group + it / n_qt; };
  auto iter_m0 = [&](int it) { return (it_lo + it % n_qt) * kQTile; };

  if (warp_idx < 4) {
    setmaxnreg_dec<24>();
    // ================================ TMA producer ================================
    if (warp_idx == 0 && lane == 0) {
      mbar_arrive_expect_tx(kv_full, 2 * S::kKVBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c) {
        tma_load_3d(sK + c * 16384, &tmap_k, kv_full, c * 64, hk, k_start + n0);
        tma_load_3d(sV + c * 16384, &tmap_v, kv_full, c * 64, hk, k_start + n0);
      }
      for (int it = 0; it < n_iter; ++it) {
        const int s = it % kQStages;
        mbar_wait(qdo_empty(s), ((it / kQStages) & 1) ^ 1);
        mbar_arrive_expect_tx(qdo_full(s), 2 * S::kQBytes);
        const int h = iter_head(it), row0 = q_start + iter_m0(it);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          tma_load_3d(sQ + s * S::kQBytes + c * kQChunk, &tmap_q, qdo_full(s), c * 64, h, row0);
          tma_load_3d(sDO + s * S::kQBytes + c * kQChunk, &tmap_do, qdo_full(s), c * 64, h, row0);
        }
      }
    }
    return;
  }

  // ================================ MMA warpgroups ================================
  setmaxnreg_inc<240>();
  const int wg = (warp_idx >> 2) - 1;
  const int tid = threadIdx.x & 127;
  const uint32_t quad = lane & 3;
  const int kr = wg * 64 + (warp_idx & 3) * 16 + (int)(lane >> 2);   // this thread's key rows in the tile: kr, kr + 8
  const float sl2 = args.scale_log2, sc = args.scale;
  float* stat = stat_all + wg * 2 * kQTile;                           // this warpgroup's copy of lse2 / delta
  const uint32_t sK_w = sK + wg * 8192, sV_w = sV + wg * 8192;        // rows [64 wg, 64 wg + 64) of every 64-column chunk
  const uint32_t sDS_w = sDS + wg * 8192;
  auto wg_sync = [&]() {   // named barrier of this warpgroup
    if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory"); else asm volatile("bar.sync 2, 128;" ::: "memory");
  };
  const bool tracing = args.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 128;
  uint32_t drop_key[2] = {0u, 0u};
  if constexpr (kDrop) {
    drop_key[0] = drop_key_part(args.drop.seed_hi, (uint32_t)(n0 + kr));
    drop_key[1] = drop_key_part(args.drop.seed_hi, (uint32_t)(n0 + kr + 8));
  }

  float dv[D / 2], dk[D / 2];
  mbar_wait(kv_full, 0);
  for (int it = 0; it < n_iter; ++it) {
    const int s = it % kQStages;
    const int h = iter_head(it), m0 = iter_m0(it);
    const uint32_t q_s = sQ + s * S::kQBytes, do_s = sDO + s * S::kQBytes;
    if (tracing && it < 64) args.trace[it * 16 + 0] = clock64();
    // row statistics of this query tile (the previous tile's readers are past their dS^T barrier)
    {
      const int row = m0 + (tid & 63);
      const bool ok = row < q_len;
      const long long off = (long long)h * args.Tq + q_start + row;
      if (tid < 64) {
        const float l = ok ? args.lse[off] : INFINITY;
        stat[tid] = (l == -INFINITY) ? INFINITY : l * 1.4426950408889634f;
      } else {
        stat[tid] = ok ? args.delta[off] : 0.f;
      }
    }
    mbar_wait(qdo_full(s), (it / kQStages) & 1);
    // ---- (a) S^T = K Q^T, (b) dP^T = V dO^T ----
    float st[kQTile / 2], dpt[kQTile / 2];
    wgmma_fence_acc(st);
    wgmma_fence_acc(dpt);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<kQTile, kBf16, 0, 0>(st, desc_kmajor_sw128(sK_w + (kk / 4) * 16384, kk % 4),
                                    desc_kmajor_sw128(q_s + (kk / 4) * kQChunk, kk % 4), kk != 0);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<kQTile, kBf16, 0, 0>(dpt, desc_kmajor_sw128(sV_w + (kk / 4) * 16384, kk % 4),
                                    desc_kmajor_sw128(do_s + (kk / 4) * kQChunk, kk % 4), kk != 0);
    wgmma_commit();
    wg_sync();            // statistics visible; every thread of the group is done with the previous dS^T tile
    wgmma_wait<0>();
    wgmma_fence_acc(st);
    wgmma_fence_acc(dpt);
    if (tracing && it < 64) args.trace[it * 16 + 1] = clock64();

    // ---- P^T = exp2(S^T * scale - LSE), dS^T = P^T o (dP^T - delta) * scale ----
    const float slope_l2 = args.alibi ? args.alibi[(long long)b * args.alibi_bs + h] * 1.4426950408889634f : 0.f;
    // interior tile: every query row of the tile sees every key of the tile -> no per-element mask
    bool interior = (m0 + kQTile <= q_len) && (n0 + kTile <= k_len);
    if (interior) {
      const int pos_first = m0 + shift, pos_last = m0 + kQTile - 1 + shift;
      const int hi_first = (wr_eff < 0) ? (k_len - 1) : min(k_len - 1, pos_first + wr_eff);
      const int lo_last = (args.wl < 0) ? 0 : max(0, pos_last - args.wl);
      interior = (hi_first >= n0 + kTile - 1) && (lo_last <= n0);
    }
    const uint32_t drop_head = kDrop ? drop_head_part(args.drop.seed_lo, (uint32_t)(b * args.Hq + h)) : 0u;
    uint32_t pfrag[kQTile / 16][4], dsfrag[kQTile / 16][4];
#pragma unroll
    for (int j = 0; j < kQTile / 8; ++j) {
      const int c = 8 * j + 2 * (int)quad;                 // query columns c, c + 1 of the tile
      const float2 l2 = *reinterpret_cast<const float2*>(stat + c);
      const float2 dl = *reinterpret_cast<const float2*>(stat + kQTile + c);
#pragma unroll
      for (int i = 0; i < 2; ++i) {                        // key rows kr, kr + 8
        const int key = n0 + kr + 8 * i;
        float p[2], ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qrow = m0 + c + e;
          float x = fmaf(st[4 * j + 2 * i + e], sl2, -(e ? l2.y : l2.x));
          if (args.alibi != nullptr) x -= slope_l2 * fabsf((float)(qrow + shift - key));
          float pe = fast_exp2(x);
          if (!interior) {
            const int pos = qrow + shift;
            const int hi = (wr_eff < 0) ? (k_len - 1) : min(k_len - 1, pos + wr_eff);
            const int lo = (args.wl < 0) ? 0 : max(0, pos - args.wl);
            pe = (key < k_len && qrow < q_len && key >= lo && key <= hi) ? pe : 0.f;
          }
          float dpe = dpt[4 * j + 2 * i + e];
          float pv = pe;
          if constexpr (kDrop) {
            // dV += (P o mask / (1-p))^T dO; d(dropped P) -> dP: the same mask and 1/(1-p)
            const bool keep = drop_keep(drop_row_part(drop_head, (uint32_t)qrow), drop_key[i], args.drop.thresh24);
            pv = keep ? pe * args.drop.rp : 0.f;
            dpe = keep ? dpe * args.drop.rp : 0.f;
          }
          p[e] = pv;
          ds[e] = pe * (dpe - (e ? dl.y : dl.x)) * sc;
        }
        pfrag[j >> 1][(j & 1) * 2 + i] = pack_h2<kBf16>(p[0], p[1]);
        const uint32_t dsp = pack_h2<kBf16>(ds[0], ds[1]);
        dsfrag[j >> 1][(j & 1) * 2 + i] = dsp;
        // dS^T -> smem row (key), 128B-swizzled: 16-byte unit j of row r lives at unit (j ^ (r & 7))
        const uint32_t r = (uint32_t)(kr + 8 * i);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sDS + r * 128u + (((uint32_t)j ^ (r & 7u)) << 4) + 4u * quad), "r"(dsp)
                     : "memory");
      }
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
    wg_sync();
    // ---- (c) dV += P^T dO, (d) dK += dS^T Q, (e) dQ = dS K over this warpgroup's keys ----
    float dq[D / 2];
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    wgmma_fence_acc(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kQTile / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(dv, pfrag[kk], desc_mnmajor_sw128(do_s, kk, kQChunk), (it | kk) != 0);
#pragma unroll
    for (int kk = 0; kk < kQTile / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(dk, dsfrag[kk], desc_mnmajor_sw128(q_s, kk, kQChunk), (it | kk) != 0);
#pragma unroll
    for (int kk = 0; kk < 64 / 16; ++kk)
      wgmma_ss<D, kBf16, 1, 1>(dq, desc_mnmajor_sw128(sDS_w, kk, 0), desc_mnmajor_sw128(sK_w, kk, 16384), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    wgmma_fence_acc(dq);
    if (tid == 0) mbar_arrive(qdo_empty(s));
    if (tracing && it < 64) args.trace[it * 16 + 2] = clock64();
    // dQ rows = queries of the tile: reduce this warpgroup's partial sums into the fp32 accumulator
    const int qr = (warp_idx & 3) * 16 + (int)(lane >> 2);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = m0 + qr + 8 * i;
      if (row >= q_len) continue;
      float* dst = args.dq_acc + ((long long)(q_start + row) * args.Hq + h) * D + 2 * quad;
#pragma unroll
      for (int j = 0; j < D / 8; ++j) red_add_v2(dst + 8 * j, dq[4 * j + 2 * i], dq[4 * j + 2 * i + 1]);
    }
  }

  // ---- epilogue: dV, dK -> bf16 / fp16 ----
  const bool vec_k = (args.dk_ts % 8 == 0) && (reinterpret_cast<uintptr_t>(args.dk) % 16 == 0);
  const bool vec_v = (args.dv_ts % 8 == 0) && (reinterpret_cast<uintptr_t>(args.dv) % 16 == 0);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = n0 + kr + 8 * i;
    const bool ok = key < k_len;
    uint16_t* pdv = args.dv + (long long)(k_start + key) * args.dv_ts + (long long)hk * D;
    uint16_t* pdk = args.dk + (long long)(k_start + key) * args.dk_ts + (long long)hk * D;
#pragma unroll
    for (int g = 0; g < D / 32; ++g) {
      uint32_t xv[4], xk[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * g + jj;
        xv[jj] = pack_h2<kBf16>(dv[4 * j + 2 * i], dv[4 * j + 2 * i + 1]);
        xk[jj] = pack_h2<kBf16>(dk[4 * j + 2 * i], dk[4 * j + 2 * i + 1]);
      }
      quad_transpose(xv, lane);
      quad_transpose(xk, lane);
      if (ok) {
        store_row8(pdv + 32 * g + 8 * quad, xv, 8, vec_v);
        store_row8(pdk + 32 * g + 8 * quad, xk, 8, vec_k);
      }
    }
  }
}

// delta[h, t] = sum_d dO[t,h,d] * O[t,h,d];  dq_acc[t,h,:] = 0.   One warp per (token, head).
template <int D, bool kBf16>
__global__ void __launch_bounds__(256)
bwd_preprocess_kernel(const uint16_t* __restrict__ o, const uint16_t* __restrict__ dout,
                      float* __restrict__ delta, float* __restrict__ dq_acc, long long Tq, int Hq, long long do_ts) {
  const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= Tq * Hq) return;
  const long long t = w / Hq;
  const int h = (int)(w % Hq);
  constexpr int kPer = D / 32;  // 4 (D=128) or 2 (D=64) elements per lane
  const uint16_t* op = o + (t * Hq + h) * D + lane * kPer;
  const uint16_t* dp = dout + t * do_ts + (long long)h * D + lane * kPer;
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; i += 2) {
    float2 a = unpack_h2<kBf16>(*reinterpret_cast<const uint32_t*>(op + i));
    float2 g = unpack_h2<kBf16>(*reinterpret_cast<const uint32_t*>(dp + i));
    acc += a.x * g.x + a.y * g.y;
  }
  acc = warp_reduce_sum(acc);
  if (lane == 0) delta[(long long)h * Tq + t] = acc;
  float* q = dq_acc + (t * Hq + h) * D + lane * kPer;
#pragma unroll
  for (int i = 0; i < kPer; ++i) q[i] = 0.f;
}

template <bool kBf16>
__global__ void __launch_bounds__(256)
bwd_convert_dq_kernel(const float* __restrict__ dq_acc, uint16_t* __restrict__ dq, long long Tq, int HD,
                      long long dq_ts) {
  const long long n = Tq * (HD / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / (HD / 4);
    const int c = (int)(i % (HD / 4)) * 4;
    float4 v = *reinterpret_cast<const float4*>(dq_acc + t * HD + c);
    uint2 o;
    o.x = pack_h2<kBf16>(v.x, v.y);
    o.y = pack_h2<kBf16>(v.z, v.w);
    *reinterpret_cast<uint2*>(dq + t * dq_ts + c) = o;
  }
}

static long long* g_bwd_trace = nullptr;
void flash_attn_bwd_set_trace(long long* p) { g_bwd_trace = p; }

static CUtensorMap make_map_thd_b(const void* base, long long tokens, int heads, int D, long long ts, bool bf16,
                                  int box_rows) {
  uint64_t dims[3] = {(uint64_t)D, (uint64_t)heads, (uint64_t)tokens};
  uint64_t strides[2] = {(uint64_t)D * 2, (uint64_t)ts * 2};
  uint32_t box[3] = {64, 1, (uint32_t)box_rows};
  return make_tensor_map(base, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, dims,
                         strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int D, bool kBf16, bool kDrop>
static cudaError_t launch_bwd(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                              const CUtensorMap& mdo, const BwdArgs& a, int num_k_tiles,
                              cudaStream_t stream) {
  using S = BwdSmem<D>;
  auto kern = flash_bwd_kernel<D, kBf16, kDrop>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid(num_k_tiles, a.Hk, a.B);
  kern<<<grid, kBwdThreads, S::kTotal, stream>>>(mq, mk, mv, mdo, a);
  return cudaGetLastError();
}

cudaError_t flash_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                           const float* lse, void* dq, void* dk, void* dv, float* dq_acc, float* delta,
                           const int* cu_q, const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D,
                           long long q_ts, long long k_ts, long long v_ts, long long do_ts, float scale, bool causal,
                           int wl, int wr, long long Tq, long long Tk, long long dq_ts, long long dk_ts,
                           long long dv_ts, int num_sms, bool is_bf16, const float* alibi_slopes,
                           int alibi_batch_stride, cudaStream_t stream) {
  return flash_attn_bwd_ex(q, k, v, o, dout, lse, dq, dk, dv, dq_acc, delta, cu_q, cu_k, B, Sq, Sk, Hq, Hk, D, q_ts, k_ts,
                           v_ts, do_ts, scale, causal, wl, wr, Tq, Tk, dq_ts, dk_ts, dv_ts, num_sms, is_bf16,
                           alibi_slopes, alibi_batch_stride, BlockView{}, 7, stream);
}

cudaError_t flash_attn_bwd_ex(const void* q, const void* k, const void* v, const void* o, const void* dout,
                              const float* lse, void* dq, void* dk, void* dv, float* dq_acc, float* delta,
                              const int* cu_q, const int* cu_k, int B, int Sq, int Sk, int Hq, int Hk, int D,
                              long long q_ts, long long k_ts, long long v_ts, long long do_ts, float scale, bool causal,
                              int wl, int wr, long long Tq, long long Tk, long long dq_ts, long long dk_ts,
                              long long dv_ts, int num_sms, bool is_bf16, const float* alibi_slopes,
                              int alibi_batch_stride, BlockView view, int phases, cudaStream_t stream) {
  if (B == 0 || Tq == 0 || Tk == 0) return cudaSuccess;
  if (D != 64 && D != 128) return cudaErrorInvalidValue;
  if (Hq % Hk != 0) return cudaErrorInvalidValue;
  // 1) delta = rowsum(dO o O), dq_acc = 0
  if (phases & 1) {
    const long long warps = Tq * Hq;
    const long long blocks = (warps * 32 + 255) / 256;
#define TB_PRE(DD, BF)                                                                                       \
  bwd_preprocess_kernel<DD, BF><<<(unsigned)blocks, 256, 0, stream>>>((const uint16_t*)o, (const uint16_t*)dout, delta, \
                                                                      dq_acc, Tq, Hq, do_ts)
    if (D == 128) { if (is_bf16) TB_PRE(128, true); else TB_PRE(128, false); }
    else { if (is_bf16) TB_PRE(64, true); else TB_PRE(64, false); }
#undef TB_PRE
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  // 2) main kernel
  cudaError_t e = cudaSuccess;
  if (phases & 2) {
  CUtensorMap mq, mk, mv, mdo;
  try {
    mq = make_map_thd_b(q, Tq, Hq, D, q_ts, is_bf16, kQTile);
    mk = make_map_thd_b(k, Tk, Hk, D, k_ts, is_bf16, kTile);
    mv = make_map_thd_b(v, Tk, Hk, D, v_ts, is_bf16, kTile);
    mdo = make_map_thd_b(dout, Tq, Hq, D, do_ts, is_bf16, kQTile);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  BwdArgs a;
  a.lse = lse; a.delta = delta; a.dq_acc = dq_acc;
  a.dk = (uint16_t*)dk; a.dv = (uint16_t*)dv;
  a.alibi = alibi_slopes; a.alibi_bs = alibi_batch_stride;
  a.cu_q = cu_q; a.cu_k = cu_k;
  a.B = B; a.Sq = Sq; a.Sk = Sk; a.Hq = Hq; a.Hk = Hk;
  a.Tq = Tq;
  a.dk_ts = dk_ts; a.dv_ts = dv_ts;
  a.scale = scale;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.causal = causal ? 1 : 0;
  a.wl = wl; a.wr = wr;
  a.trace = g_bwd_trace;
  a.q_bs = view.q_bs > 0 ? view.q_bs : Sq; a.q_off = view.q_off;
  a.k_bs = view.k_bs > 0 ? view.k_bs : Sk; a.k_off = view.k_off;
  const int max_k = cu_k ? (int)Tk : Sk;
  const int num_k_tiles = (max_k + kTile - 1) / kTile;
  const bool drop = view.p_drop > 0.f;
  if (drop) {
    if (view.p_drop >= 1.f) return cudaErrorInvalidValue;
    a.drop.thresh24 = (uint32_t)((double)view.p_drop * 16777216.0 + 0.5);   // mirrored in dropout_keep_mask
    a.drop.rp = 1.f / (1.f - view.p_drop);
    a.drop.seed_lo = (uint32_t)(view.seed & 0xffffffffull);
    a.drop.seed_hi = (uint32_t)(view.seed >> 32);
  } else {
    a.drop = DropoutParams{0u, 1.f, 0u, 0u};
  }
#define TB_BWD(DD, BF)                                                                            \
  (drop ? launch_bwd<DD, BF, true>(mq, mk, mv, mdo, a, num_k_tiles, stream)                  \
        : launch_bwd<DD, BF, false>(mq, mk, mv, mdo, a, num_k_tiles, stream))
  if (is_bf16) e = (D == 128) ? TB_BWD(128, true) : TB_BWD(64, true);
  else e = (D == 128) ? TB_BWD(128, false) : TB_BWD(64, false);
#undef TB_BWD
  if (e != cudaSuccess) return e;
  }
  // 3) dq = bf16(dq_acc)
  if (phases & 4) {
    const long long n = Tq * (long long)(Hq * D / 4);
    long long blocks = (n + 255) / 256;
    if (blocks > (long long)num_sms * 16) blocks = (long long)num_sms * 16;
    if (is_bf16) bwd_convert_dq_kernel<true><<<(unsigned)blocks, 256, 0, stream>>>(dq_acc, (uint16_t*)dq, Tq, Hq * D, dq_ts);
    else bwd_convert_dq_kernel<false><<<(unsigned)blocks, 256, 0, stream>>>(dq_acc, (uint16_t*)dq, Tq, Hq * D, dq_ts);
    e = cudaGetLastError();
  }
  return e;
}

}  // namespace tb
