// FlashAttention backward on wgmma / TMA for sm_90a.
//
// One CTA per (128-key tile, kv head, batch); it loops over the q heads of the GQA group and over the query tiles that
// can see this key tile, so dK/dV are accumulated in registers with no atomics.  Query tiles have 128 rows at D = 64
// and 64 rows at D = 128 (there the 64-register dK and dV accumulators leave no room for 128-column S^T / dP^T tiles)
// or with dropout (bwd_q_tile).
// Two MMA warpgroups own 64 keys each.  The score tile is computed TRANSPOSED (S^T = K Q^T: accumulator rows = keys,
// columns = queries), which lets every later GEMM take its operands in place:
//   (a) S^T  = K  Q^T    A = K  (smem, K-major)          B = Q  (smem, K-major)
//   (b) dP^T = V  dO^T   A = V  (smem, K-major)          B = dO (smem, K-major)
//   in registers:  P^T = exp2(S^T*scale - LSE), dS^T = P^T o (dP^T - delta) * scale
//   (c) dV  += P^T dO    A = P^T  (registers)            B = dO (smem, MN-major)
//   (d) dK  += dS^T Q    A = dS^T (registers)            B = Q  (smem, MN-major)
//   (e) dQ   = dS K      A = dS^T (smem, read MN-major)  B = K  (smem, MN-major), over all 128 keys of the CTA
// Step (e) reads the dS^T rows of both warpgroups, so it waits on a barrier of the two; each warpgroup then computes a
// 64 x 64 dQ tile (its half of the query rows at D = 64, its half of the columns at D = 128; with 64-row tiles at
// D = 64, the partial sum over its own 64 keys), stages it in shared memory while its dV / dK MMAs run, and one thread
// adds it to the fp32 accumulator with a TMA bulk reduce-add (double-buffered staging).
// Query rows past the end of the sequence have P = dS = 0, so their rows of the tile add exact zeros.
// Q/dO tiles stream through a 2-stage TMA ring; K/V stay resident.
// The deterministic backward compiles step (e) out and computes dQ with flash_bwd_dq_kernel (below) instead.
//
// Reference parity: FA2 backward reached by reference torchacc/ops/flash_attn.py:56,152,206,252,301.
#include <math.h>
#include <stdio.h>

#include <type_traits>

#include "../common/ptx.cuh"
#include "common.cuh"
#include "mask.cuh"

namespace tb {

constexpr int kTile = 128;        // keys per CTA
constexpr int kBwdThreads = 384;  // producer warpgroup + 2 MMA warpgroups (64 keys each)
constexpr int kQStages = 2;
// Query rows per iteration: 128 at D = 64 without dropout.  With dropout the mask state does not fit next to the
// 128-column S^T / dP^T tiles without spills (the kDQ = false kernel), and the default and deterministic kernels must
// share the tile so that their dK / dV stay bitwise equal, so both use 64 rows.
constexpr int bwd_q_tile(int D, bool drop) { return (D == 64 && !drop) ? 128 : 64; }

// Phase profile of the main kernel (kProf instantiations, attn_bwd_set_profile): for the CTAs of kv head 0, sequence
// 0 and key tiles [0, prof_ctas), one elected thread per role writes clock64() stamps into a record of kProfCtaWords
// u64 at prof + blockIdx.x * kProfCtaWords:
//   [0] n_iter  [1] %smid  [2] CTA start  [3] K/V landed  [4] / [5] MMA warpgroup 0 / 1 done  [6] producer done
//   [kProfHead + it * kProfSlots + ...] for iterations it < kProfIters:
//     [0, kProfWgSlots) warpgroup 0 phase ends, [kProfWgSlots, 2 kProfWgSlots) warpgroup 1, then the producer's
//     empty-wait done and stage issued.  Phase order: benchmarks/attn_bwd_phases.py.
constexpr int kProfHead = 8, kProfWgSlots = 10, kProfSlots = 2 * kProfWgSlots + 2, kProfIters = 256;
constexpr long long kProfCtaWords = kProfHead + (long long)kProfIters * kProfSlots;

struct BwdArgs : AttnShape {
  const float* lse;
  const float* delta;
  uint16_t* dk;                // bf16 or fp16 (kernel template)
  uint16_t* dv;
  long long dk_ts, dv_ts;
  unsigned long long* prof;    // kProf only
  long long prof_ctas;
};

__device__ __forceinline__ unsigned long long prof_clock() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
  return t;
}
__device__ __forceinline__ unsigned long long smid() {
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

template <int D, bool kDrop>
struct BwdSmem {
  static constexpr int kQTile = bwd_q_tile(D, kDrop);
  static constexpr int kChunks = D / 64;
  static constexpr int kKVBytes = kTile * D * 2;
  static constexpr int kQBytes = kQTile * D * 2;
  static constexpr int kDQBytes = 64 * 64 * 4;              // one warpgroup's fp32 dQ tile
  static constexpr int kK = 0;
  static constexpr int kV = kK + kKVBytes;
  static constexpr int kQ = kV + kKVBytes;
  static constexpr int kDO = kQ + kQStages * kQBytes;
  static constexpr int kDS = kDO + kQStages * kQBytes;      // dS^T: kQTile / 64 chunks of [128 keys][64 queries]
  static constexpr int kDQ = kDS + kTile * kQTile * 2;      // dQ staging [2 buffers][2 warpgroups], 1024-aligned
  static constexpr int kStat = kDQ + 2 * 2 * kDQBytes;      // per warpgroup: lse2[kQTile], delta[kQTile]
  static constexpr int kBar = kStat + 2 * 2 * kQTile * 4;
  static constexpr int kTotal = kBar + 128 + 1024;
  static_assert(kTotal <= 227 * 1024, "backward shared memory exceeds the sm_90 limit");
};

// kDQ = false drops step (e) -- the dS^T stores, the dQ MMA and the reduce-adds -- and leaves dK / dV only; the
// deterministic backward computes dQ afterwards in flash_bwd_dq_kernel.
// kProf = true adds the phase stamps described at kProfHead.
template <int D, bool kBf16, bool kDrop, bool kDQ, bool kProf = false>
__global__ void __launch_bounds__(kBwdThreads, 1)
flash_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                 const __grid_constant__ CUtensorMap tmap_dq, const BwdArgs args) {
  using S = BwdSmem<D, kDrop>;
  constexpr int kChunks = S::kChunks;
  constexpr int kQTile = S::kQTile;
  constexpr int kQChunk = kQTile * 128;   // bytes of one 64-column chunk of a Q / dO stage

  unsigned long long t_start = 0;
  if constexpr (kProf) t_start = prof_clock();
  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();
  const int b = blockIdx.z, hk = blockIdx.y, jt = blockIdx.x;
  const int group = args.Hq / args.Hk;
  int q_start, q_len, k_start, k_len;
  seq_bounds(args, b, q_start, q_len, k_start, k_len);
  const int n0 = jt * kTile;
  if (n0 >= k_len) return;

  int it_lo, n_qt;
  query_tile_range(n0, kTile, q_len, k_len, args.wl, args.wr, kQTile, it_lo, n_qt);
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
  const uint32_t sDQ = base + S::kDQ;
  float* stat_all = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + S::kStat);
  const uint32_t bar = base + S::kBar;
  const uint32_t kv_full = bar;
  auto qdo_full = [&](int s) { return bar + 8u * (1 + s); };
  auto qdo_empty = [&](int s) { return bar + 8u * (1 + kQStages + s); };

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v); tma_prefetch_desc(&tmap_do);
    if constexpr (kDQ) tma_prefetch_desc(&tmap_dq);
  }
  if (warp_idx == 1 && lane == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < kQStages; ++s) { mbar_init(qdo_full(s), 1); mbar_init(qdo_empty(s), 2); }
    fence_mbar_init();
  }
  __syncthreads();

  // this CTA's phase record, or null
  unsigned long long* prof = nullptr;
  if constexpr (kProf) {
    if (b == 0 && hk == 0 && jt < args.prof_ctas) prof = args.prof + (long long)jt * kProfCtaWords;
    if (prof != nullptr && threadIdx.x == 0) {
      prof[0] = (unsigned long long)n_iter;
      prof[1] = smid();
      prof[2] = t_start;
    }
  }
  // stamp slot `slot` of iteration `it` (one elected thread per role calls it)
  auto stamp = [&](int it, int slot) {
    if constexpr (kProf) {
      if (prof != nullptr && it < kProfIters) prof[kProfHead + it * kProfSlots + slot] = prof_clock();
    }
  };

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
        stamp(it, 2 * kProfWgSlots);
        mbar_arrive_expect_tx(qdo_full(s), 2 * S::kQBytes);
        const int h = iter_head(it), row0 = q_start + iter_m0(it);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          tma_load_3d(sQ + s * S::kQBytes + c * kQChunk, &tmap_q, qdo_full(s), c * 64, h, row0);
          tma_load_3d(sDO + s * S::kQBytes + c * kQChunk, &tmap_do, qdo_full(s), c * 64, h, row0);
        }
        stamp(it, 2 * kProfWgSlots + 1);
      }
      if constexpr (kProf) {
        if (prof != nullptr) prof[6] = prof_clock();
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
  // step (e) of this warpgroup: dQ rows [dq_row0, +64) of the query tile, columns [dq_col0, +64), over all 128 keys;
  // a 64 x 64 tile has nothing to split, so there each warpgroup adds the partial sum over its own 64 keys
  constexpr bool kDqOwnKeys = kQTile == 64 && D == 64;
  const int dq_row0 = kQTile == 128 ? 64 * wg : 0, dq_col0 = D == 128 ? 64 * wg : 0;
  const uint32_t dq_a = sDS + (dq_row0 / 64) * 16384 + (kDqOwnKeys ? wg * 8192 : 0);   // dS^T chunk (and key rows)
  const uint32_t dq_b = sK + (dq_col0 / 64) * 16384 + (kDqOwnKeys ? wg * 8192 : 0);    // K chunk (and key rows)
  auto wg_sync = [&]() {   // named barrier of this warpgroup
    if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory"); else asm volatile("bar.sync 2, 128;" ::: "memory");
  };
  auto mma_sync = [&]() {  // named barrier of both MMA warpgroups: step (e) reads the other warpgroup's dS^T rows
    if constexpr (kDQ) asm volatile("bar.sync 3, 256;" ::: "memory"); else wg_sync();
  };
  uint32_t drop_key[2] = {0u, 0u};
  if constexpr (kDrop) {
    drop_key[0] = drop_key_part(args.drop.seed_hi, (uint32_t)(n0 + kr));
    drop_key[1] = drop_key_part(args.drop.seed_hi, (uint32_t)(n0 + kr + 8));
  }

  const int wslot = wg * kProfWgSlots;
  auto mark = [&](int it, int slot) { if (tid == 0) stamp(it, wslot + slot); };   // phase ends of this warpgroup

  float dv[D / 2], dk[D / 2];
  mbar_wait(kv_full, 0);
  if constexpr (kProf) {
    if (prof != nullptr && threadIdx.x == 128) prof[3] = prof_clock();
  }
  for (int it = 0; it < n_iter; ++it) {
    const int s = it % kQStages;
    const int h = iter_head(it), m0 = iter_m0(it);
    const uint32_t q_s = sQ + s * S::kQBytes, do_s = sDO + s * S::kQBytes;
    mbar_wait(qdo_full(s), (it / kQStages) & 1);
    mark(it, 0);
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
    mark(it, 1);
    // row statistics of this query tile, loaded while the MMAs run (the previous tile's readers are past their dS^T
    // barrier)
#pragma unroll
    for (int r = tid; r < 2 * kQTile; r += 128) {   // stat[0, kQTile): lse2, stat[kQTile, 2 kQTile): delta
      const int row = m0 + (r & (kQTile - 1));
      const bool ok = row < q_len;
      const long long off = (long long)h * args.Tq + q_start + row;
      if (r < kQTile) {
        const float l = ok ? args.lse[off] : INFINITY;
        stat[r] = (l == -INFINITY) ? INFINITY : l * 1.4426950408889634f;
      } else {
        stat[r] = ok ? args.delta[off] : 0.f;
      }
    }
    mark(it, 2);
    mma_sync();           // statistics visible; every reader of the previous dS^T tile is done with it
    mark(it, 3);
    wgmma_wait<0>();
    wgmma_fence_acc(st);
    wgmma_fence_acc(dpt);
    mark(it, 4);

    // ---- P^T = exp2(S^T * scale - LSE), dS^T = P^T o (dP^T - delta) * scale ----
    const float slope_l2 = args.alibi ? args.alibi[(long long)b * args.alibi_bs + h] * 1.4426950408889634f : 0.f;
    const bool interior = tile_interior(m0, kQTile, n0, kTile, q_len, k_len, args.wl, args.wr);
    const uint32_t drop_head = kDrop ? drop_head_part(args.drop.seed_lo, (uint32_t)(b * args.Hq + h)) : 0u;
    uint32_t pfrag[kQTile / 16][4], dsfrag[kQTile / 16][4];
    // kMasked = false: an interior tile without ALiBi, where P^T is exp2 alone.  The test is uniform over the tile, so
    // it is taken once here: folded into the loop, the compiler predicates the mask and ALiBi arithmetic and every
    // element pays for it.
    auto softmax_bwd = [&](auto masked) {
      constexpr bool kMasked = decltype(masked)::value;
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
            if (kMasked && args.alibi != nullptr) x -= slope_l2 * fabsf((float)(qrow + (k_len - q_len) - key));
            float pe = fast_exp2(x);
            if (kMasked && !interior) {
              int lo, hi;   // hi <= k_len - 1: keys past the sequence are invisible
              key_bounds(qrow, q_len, k_len, args.wl, args.wr, lo, hi);
              pe = (qrow < q_len && key >= lo && key <= hi) ? pe : 0.f;
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
          if constexpr (kDQ) {
            // dS^T -> smem row (key) of chunk j / 8, 128B-swizzled: 16-byte unit u of row r lives at unit (u ^ (r & 7))
            const uint32_t r = (uint32_t)(kr + 8 * i), u = (uint32_t)j & 7u;
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sDS + (j >> 3) * 16384 + r * 128u + ((u ^ (r & 7u)) << 4) +
                                                            4u * quad),
                         "r"(dsp)
                         : "memory");
          }
        }
      }
    };
    if (interior && args.alibi == nullptr) softmax_bwd(std::false_type{});
    else softmax_bwd(std::true_type{});
    if constexpr (kDQ) {
      fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      // the reduce-add issued two tiles ago has read the staging buffer this tile writes (ordered by the barrier)
      if (tid == 0) tma_store_wait_read<1>();
    }
    mark(it, 5);
    mma_sync();
    mark(it, 6);
    // ---- (e) dQ = dS K, then (c) dV += P^T dO, (d) dK += dS^T Q: dQ is its own group, so the dQ tile is staged and
    // reduced while the tensor cores work on dV / dK ----
    float dq[kDQ ? 32 : 1];
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    if constexpr (kDQ) wgmma_fence_acc(dq);
    wgmma_fence();
    if constexpr (kDQ) {
#pragma unroll
      for (int kk = 0; kk < (kDqOwnKeys ? 64 : kTile) / 16; ++kk)
        wgmma_ss<64, kBf16, 1, 1>(dq, desc_mnmajor_sw128(dq_a, kk, 0), desc_mnmajor_sw128(dq_b, kk, 0), kk != 0);
      wgmma_commit();
    }
#pragma unroll
    for (int kk = 0; kk < kQTile / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(dv, pfrag[kk], desc_mnmajor_sw128(do_s, kk, kQChunk), (it | kk) != 0);
#pragma unroll
    for (int kk = 0; kk < kQTile / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(dk, dsfrag[kk], desc_mnmajor_sw128(q_s, kk, kQChunk), (it | kk) != 0);
    wgmma_commit();
    mark(it, 7);
    if constexpr (kDQ) {
      wgmma_wait<1>();
      wgmma_fence_acc(dq);
      // dQ tile -> staging buffer as two [64 rows][32 fp32] halves, 128B-swizzled like the TMA box, then one bulk
      // reduce-add per half into dq_acc.  Rows past the end of dq_acc are clipped by the tensor map.
      const uint32_t stg = sDQ + ((it & 1) * 2 + wg) * S::kDQBytes;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t r = (warp_idx & 3) * 16 + (lane >> 2) + 8 * i;
#pragma unroll
        for (int j = 0; j < 8; ++j) {   // columns 8 j + 2 quad, + 1
          const uint32_t u = 2 * (j & 3) + (quad >> 1);
          const uint32_t addr = stg + (j >> 2) * 8192 + r * 128 + ((u ^ (r & 7)) << 4) + (quad & 1) * 8;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(dq[4 * j + 2 * i]), "f"(dq[4 * j + 2 * i + 1])
                       : "memory");
        }
      }
      fence_proxy_async_smem();
      wg_sync();
      if (tid == 0) {
        const int row = q_start + m0 + dq_row0;
        tma_reduce_add_3d(&tmap_dq, stg, dq_col0, h, row);
        tma_reduce_add_3d(&tmap_dq, stg + 8192, dq_col0 + 32, h, row);
        tma_store_commit();
      }
      mark(it, 8);
    }
    wgmma_wait<0>();
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    mark(it, 9);
    if (tid == 0) mbar_arrive(qdo_empty(s));
  }
  if constexpr (kProf) {
    if (prof != nullptr && tid == 0) prof[4 + wg] = prof_clock();
  }
  if constexpr (kDQ) {
    if (tid == 0) tma_store_wait<0>();   // staging buffers stay allocated until the reduce-adds have completed
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

// ================================ deterministic dQ ================================
// Query-stationary dQ = sum over key tiles of dS K, with the forward kernel's shape: one CTA per (128 query rows, q head,
// sequence), a TMA producer warpgroup (Q and dO once, K and V through 2-stage rings) and two MMA warpgroups of 64 rows.
// Per key tile:
//   S  = Q  K^T    A = Q  (smem, K-major)     B = K (smem, K-major)
//   dP = dO V^T    A = dO (smem, K-major)     B = V (smem, K-major)
//   in registers:  P = exp2(S*scale*log2e - LSE*log2e), dS = P o (dP - delta) * scale
//   dQ += dS K     A = dS (registers)         B = K (smem, MN-major)
// Every dQ row is owned by one thread quad and accumulated over the key tiles in a fixed order, so the result does not
// depend on scheduling: no atomics, no fp32 workspace, no semaphores.  Register budget at D = 128 with 128-key tiles:
// the S, dP and dQ accumulators (3 x 64 fp32) plus the dS fragments fit the 240 registers of an MMA warpgroup without
// spills (check with -Xptxas -v after changing the tile; 64-key tiles are the fallback if they stop fitting).
constexpr int kDqRows = 128;   // query rows per CTA (64 per MMA warpgroup)
constexpr int kDqKeys = 128;   // keys per K / V tile
constexpr int kDqStages = 2;

struct DqArgs : AttnShape {
  const float* lse;
  const float* delta;
  uint16_t* dq;                // bf16 or fp16 (kernel template)
  long long dq_ts;
  int num_q_tiles;
};

template <int D>
struct DqSmem {
  static constexpr int kQBytes = kDqRows * D * 2;     // Q / dO: D/64 chunks of [128 rows][64 columns]
  static constexpr int kKBytes = kDqKeys * D * 2;     // one K or V stage: D/64 chunks of [64 keys][64 columns]
  static constexpr int kQ = 0;
  static constexpr int kDO = kQ + kQBytes;
  static constexpr int kK = kDO + kQBytes;
  static constexpr int kV = kK + kDqStages * kKBytes;
  static constexpr int kBar = kV + kDqStages * kKBytes;
  static constexpr int kTotal = kBar + 128 + 1024;
};

template <int D, bool kBf16, bool kDrop>
__global__ void __launch_bounds__(kBwdThreads, 1)
flash_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                    const DqArgs args) {
  using S = DqSmem<D>;
  constexpr int kChunks = D / 64;
  constexpr int kQChunk = kDqRows * 128;   // bytes of one 64-column chunk of Q / dO
  constexpr int kKChunk = kDqKeys * 128;   // bytes of one 64-column chunk of a K / V stage

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();
  const int b = blockIdx.z, h = blockIdx.y;
  const int hk = h / (args.Hq / args.Hk);
  const int tile = args.num_q_tiles - 1 - (int)blockIdx.x;  // heavy (late) causal tiles first
  int q_start, q_len, k_start, k_len;
  seq_bounds(args, b, q_start, q_len, k_start, k_len);
  const int m0 = tile * kDqRows;
  if (m0 >= q_len) return;

  int j_lo, n_tiles;
  key_tile_range(m0, kDqRows, q_len, k_len, args.wl, args.wr, kDqKeys, j_lo, n_tiles);
  if (n_tiles <= 0) {  // no key visible to these rows: dQ = 0
    for (int r = threadIdx.x; r < min(kDqRows, q_len - m0); r += blockDim.x) {
      uint16_t* p = args.dq + (long long)(q_start + m0 + r) * args.dq_ts + (long long)h * D;
      for (int d = 0; d < D; ++d) p[d] = 0;
    }
    return;
  }

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base + S::kQ, sDO = base + S::kDO, sK = base + S::kK, sV = base + S::kV;
  const uint32_t bar = base + S::kBar;
  const uint32_t q_full = bar;
  auto kv_full = [&](int s) { return bar + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar + 8u * (1 + kDqStages + s); };

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v); tma_prefetch_desc(&tmap_do);
  }
  if (warp_idx == 1 && lane == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kDqStages; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 2); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    setmaxnreg_dec<24>();
    // ================================ TMA producer ================================
    if (warp_idx == 0 && lane == 0) {
      mbar_arrive_expect_tx(q_full, 2 * S::kQBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c) {
        tma_load_3d(sQ + c * kQChunk, &tmap_q, q_full, c * 64, h, q_start + m0);
        tma_load_3d(sDO + c * kQChunk, &tmap_do, q_full, c * 64, h, q_start + m0);
      }
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % kDqStages;
        const int tok = k_start + (j_lo + t) * kDqKeys;
        mbar_wait(kv_empty(s), ((t / kDqStages) & 1) ^ 1);
        mbar_arrive_expect_tx(kv_full(s), 2 * S::kKBytes);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          tma_load_3d(sK + s * S::kKBytes + c * kKChunk, &tmap_k, kv_full(s), c * 64, hk, tok);
          tma_load_3d(sV + s * S::kKBytes + c * kKChunk, &tmap_v, kv_full(s), c * 64, hk, tok);
        }
      }
    }
    return;
  }

  // ================================ MMA warpgroups ================================
  setmaxnreg_inc<240>();
  const int wg = (warp_idx >> 2) - 1;
  const uint32_t quad = lane & 3;
  const int r0 = wg * 64 + (warp_idx & 3) * 16 + (int)(lane >> 2);   // this thread's rows inside the tile: r0, r0 + 8
  const bool elected = (threadIdx.x & 127) == 0;
  int lo[2], hi[2], pos_q[2];
  uint32_t drop_row[2] = {0u, 0u};
  float lse2[2], dlt[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = min(m0 + r0 + 8 * i, q_len - 1);
    key_bounds(row, q_len, k_len, args.wl, args.wr, lo[i], hi[i]);
    pos_q[i] = row + (k_len - q_len);
    if constexpr (kDrop)
      drop_row[i] = drop_row_part(drop_head_part(args.drop.seed_lo, (uint32_t)(b * args.Hq + h)), (uint32_t)(m0 + r0 + 8 * i));
    // row statistics; rows past the sequence get LSE = +inf, i.e. P = 0 (so do fully masked rows, LSE = -inf)
    const bool ok = m0 + r0 + 8 * i < q_len;
    const long long off = (long long)h * args.Tq + q_start + m0 + r0 + 8 * i;
    const float l = ok ? args.lse[off] : INFINITY;
    lse2[i] = (l == -INFINITY) ? INFINITY : l * 1.4426950408889634f;
    dlt[i] = ok ? args.delta[off] : 0.f;
  }
  const bool has_alibi = args.alibi != nullptr;
  const float slope_l2 = has_alibi ? args.alibi[(long long)b * args.alibi_bs + h] * 1.4426950408889634f : 0.f;
  const float sl2 = has_alibi ? 1.f : args.scale_log2;   // mask_score_tile has scaled the ALiBi scores already
  const uint32_t wq = wg * 8192;                          // this warpgroup's 64 rows inside a Q / dO chunk

  float dq[D / 2];
  mbar_wait(q_full, 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int s = t % kDqStages;
    const int n0 = (j_lo + t) * kDqKeys;
    const uint32_t k_s = sK + s * S::kKBytes, v_s = sV + s * S::kKBytes;
    mbar_wait(kv_full(s), (t / kDqStages) & 1);
    // ---- S = Q K^T, dP = dO V^T ----
    float sacc[kDqKeys / 2], dpacc[kDqKeys / 2];
    wgmma_fence_acc(sacc);
    wgmma_fence_acc(dpacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<kDqKeys, kBf16, 0, 0>(sacc, desc_kmajor_sw128(sQ + (kk / 4) * kQChunk + wq, kk % 4),
                                     desc_kmajor_sw128(k_s + (kk / 4) * kKChunk, kk % 4), kk != 0);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<kDqKeys, kBf16, 0, 0>(dpacc, desc_kmajor_sw128(sDO + (kk / 4) * kQChunk + wq, kk % 4),
                                     desc_kmajor_sw128(v_s + (kk / 4) * kKChunk, kk % 4), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sacc);
    wgmma_fence_acc(dpacc);

    // ---- P = exp2(S * scale - LSE) (masked entries: -inf -> 0), dS = P o (dP - delta) * scale ----
    mask_score_tile<kDqKeys>(sacc, n0, quad, lo, hi, pos_q, has_alibi, args.scale_log2, slope_l2);
    uint32_t dsfrag[kDqKeys / 16][4];
#pragma unroll
    for (int j = 0; j < kDqKeys / 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = fast_exp2(fmaf(sacc[4 * j + 2 * i + e], sl2, -lse2[i]));
          float dp = dpacc[4 * j + 2 * i + e];
          if constexpr (kDrop) {
            // d(dropped P) -> dP: the forward's mask and 1/(1-p)
            const uint32_t key = (uint32_t)(n0 + 8 * j + 2 * (int)quad + e);
            dp = drop_keep(drop_row[i], drop_key_part(args.drop.seed_hi, key), args.drop.thresh24) ? dp * args.drop.rp
                                                                                                   : 0.f;
          }
          ds[e] = p * (dp - dlt[i]) * args.scale;
        }
        dsfrag[j >> 1][(j & 1) * 2 + i] = pack_h2<kBf16>(ds[0], ds[1]);
      }
    // ---- dQ += dS K ----
    wgmma_fence_acc(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kDqKeys / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(dq, dsfrag[kk], desc_mnmajor_sw128(k_s, kk, kKChunk), (t | kk) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dq);
    if (elected) mbar_arrive(kv_empty(s));
  }

  // ---- epilogue: dQ -> bf16 / fp16 ----
  const bool vec = (args.dq_ts % 8 == 0) && (reinterpret_cast<uintptr_t>(args.dq) % 16 == 0);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = m0 + r0 + 8 * i;
    const bool valid = row < q_len;
    uint16_t* p = args.dq + (long long)(q_start + row) * args.dq_ts + (long long)h * D;
#pragma unroll
    for (int g = 0; g < D / 32; ++g) {
      uint32_t x[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * g + jj;
        x[jj] = pack_h2<kBf16>(dq[4 * j + 2 * i], dq[4 * j + 2 * i + 1]);
      }
      quad_transpose(x, lane);
      if (valid) store_row8(p + 32 * g + 8 * quad, x, 8, vec);
    }
  }
}

// delta[h, t] = sum_d dO[t,h,d] * O[t,h,d];  dq_acc[t,h,:] = 0 (when given).   One warp per (token, head).
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
  if (dq_acc == nullptr) return;   // deterministic backward: dQ is written by flash_bwd_dq_kernel
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

// fp32 dQ accumulator [tokens, heads, D]: reduce-add boxes of 64 rows x 32 columns (128 bytes), 128B-swizzled
static CUtensorMap make_map_dq_acc(float* acc, long long tokens, int heads, int D) {
  uint64_t dims[3] = {(uint64_t)D, (uint64_t)heads, (uint64_t)tokens};
  uint64_t strides[2] = {(uint64_t)D * 4, (uint64_t)heads * D * 4};
  uint32_t box[3] = {32, 1, 64};
  return make_tensor_map(acc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int D, bool kBf16, bool kDrop, bool kDQ, bool kProf = false>
static cudaError_t launch_bwd(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                              const CUtensorMap& mdo, const CUtensorMap& mdq, const BwdArgs& a, int num_k_tiles,
                              cudaStream_t stream) {
  using S = BwdSmem<D, kDrop>;
  auto kern = flash_bwd_kernel<D, kBf16, kDrop, kDQ, kProf>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid(num_k_tiles, a.Hk, a.B);
  kern<<<grid, kBwdThreads, S::kTotal, stream>>>(mq, mk, mv, mdo, mdq, a);
  return cudaGetLastError();
}

template <int D, bool kBf16, bool kDrop>
static cudaError_t launch_bwd_dq(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                 const CUtensorMap& mdo, const DqArgs& a, cudaStream_t stream) {
  using S = DqSmem<D>;
  auto kern = flash_bwd_dq_kernel<D, kBf16, kDrop>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid(a.num_q_tiles, a.Hq, a.B);
  kern<<<grid, kBwdThreads, S::kTotal, stream>>>(mq, mk, mv, mdo, a);
  return cudaGetLastError();
}

// phase-profile buffer of the next main-kernel launches (attn_bwd_set_profile), null: profiling off
static unsigned long long* g_prof = nullptr;
static long long g_prof_ctas = 0;

long long attn_bwd_set_profile(unsigned long long* buf, long long ctas) {
  g_prof = buf;
  g_prof_ctas = buf != nullptr ? ctas : 0;
  return kProfCtaWords;
}

cudaError_t flash_attn_bwd(const AttnParams& p, int num_sms, cudaStream_t stream) {
  if (p.B == 0 || p.Tq == 0 || p.Tk == 0) return cudaSuccess;
  AttnShape shape;
  cudaError_t e = make_shape(p, shape);
  if (e != cudaSuccess) return e;
  const int D = p.D, Hq = p.Hq;
  const long long Tq = p.Tq;
  const bool is_bf16 = p.is_bf16, drop = p.p_drop > 0.f, deterministic = p.deterministic;
  // 1) delta = rowsum(dO o O), dq_acc = 0 (the deterministic path has no accumulator)
  if (p.phases & 1) {
    float* acc = deterministic ? nullptr : p.dq_acc;
    const long long warps = Tq * Hq;
    const long long blocks = (warps * 32 + 255) / 256;
#define TB_PRE(DD, BF)                                                                                              \
  bwd_preprocess_kernel<DD, BF><<<(unsigned)blocks, 256, 0, stream>>>((const uint16_t*)p.o, (const uint16_t*)p.dout, \
                                                                      p.delta, acc, Tq, Hq, p.do_ts)
    if (D == 128) { if (is_bf16) TB_PRE(128, true); else TB_PRE(128, false); }
    else { if (is_bf16) TB_PRE(64, true); else TB_PRE(64, false); }
#undef TB_PRE
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  // 2) main kernel: dK / dV (+ dQ reduce-added into dq_acc unless deterministic)
  if (p.phases & 2) {
  CUtensorMap mq, mk, mv, mdo, mdq;
  try {
    mq = make_map_thd(p.q, Tq, Hq, D, p.q_ts, is_bf16, bwd_q_tile(D, drop));
    mk = make_map_thd(p.k, p.Tk, p.Hk, D, p.k_ts, is_bf16, kTile);
    mv = make_map_thd(p.v, p.Tk, p.Hk, D, p.v_ts, is_bf16, kTile);
    mdo = make_map_thd(p.dout, Tq, Hq, D, p.do_ts, is_bf16, bwd_q_tile(D, drop));
    mdq = deterministic ? mq : make_map_dq_acc(p.dq_acc, Tq, Hq, D);   // unused by the deterministic kernel
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  BwdArgs a;
  static_cast<AttnShape&>(a) = shape;
  a.lse = p.lse; a.delta = p.delta;
  a.dk = (uint16_t*)p.dk; a.dv = (uint16_t*)p.dv;
  a.dk_ts = p.dk_ts; a.dv_ts = p.dv_ts;
  a.prof = g_prof; a.prof_ctas = g_prof_ctas;
  const int max_k = p.cu_k ? (int)p.Tk : p.Sk;
  const int num_k_tiles = (max_k + kTile - 1) / kTile;
#define TB_BWD(DD, BF, DQ)                                                                        \
  (drop ? launch_bwd<DD, BF, true, DQ>(mq, mk, mv, mdo, mdq, a, num_k_tiles, stream)         \
        : launch_bwd<DD, BF, false, DQ>(mq, mk, mv, mdo, mdq, a, num_k_tiles, stream))
  if (g_prof != nullptr && D == 64 && is_bf16 && !drop) {   // the profiled instantiations: the flagship's only
    e = deterministic ? launch_bwd<64, true, false, false, true>(mq, mk, mv, mdo, mdq, a, num_k_tiles, stream)
                      : launch_bwd<64, true, false, true, true>(mq, mk, mv, mdo, mdq, a, num_k_tiles, stream);
  } else if (!deterministic) {
    if (is_bf16) e = (D == 128) ? TB_BWD(128, true, true) : TB_BWD(64, true, true);
    else e = (D == 128) ? TB_BWD(128, false, true) : TB_BWD(64, false, true);
  } else {
    if (is_bf16) e = (D == 128) ? TB_BWD(128, true, false) : TB_BWD(64, true, false);
    else e = (D == 128) ? TB_BWD(128, false, false) : TB_BWD(64, false, false);
  }
#undef TB_BWD
  if (e != cudaSuccess) return e;
  }
  // 3) dq = cast(dq_acc), or the deterministic dQ kernel
  if ((p.phases & 4) && !deterministic) {
    const long long n = Tq * (long long)(Hq * D / 4);
    long long blocks = (n + 255) / 256;
    if (blocks > (long long)num_sms * 16) blocks = (long long)num_sms * 16;
    if (is_bf16) bwd_convert_dq_kernel<true><<<(unsigned)blocks, 256, 0, stream>>>(p.dq_acc, (uint16_t*)p.dq, Tq, Hq * D, p.dq_ts);
    else bwd_convert_dq_kernel<false><<<(unsigned)blocks, 256, 0, stream>>>(p.dq_acc, (uint16_t*)p.dq, Tq, Hq * D, p.dq_ts);
    e = cudaGetLastError();
  } else if (p.phases & 4) {
    CUtensorMap mq, mk, mv, mdo;
    try {
      mq = make_map_thd(p.q, Tq, Hq, D, p.q_ts, is_bf16, kDqRows);
      mk = make_map_thd(p.k, p.Tk, p.Hk, D, p.k_ts, is_bf16, kDqKeys);
      mv = make_map_thd(p.v, p.Tk, p.Hk, D, p.v_ts, is_bf16, kDqKeys);
      mdo = make_map_thd(p.dout, Tq, Hq, D, p.do_ts, is_bf16, kDqRows);
    } catch (const std::exception& e) {
      fprintf(stderr, "%s\n", e.what());
      return cudaErrorInvalidValue;
    }
    DqArgs a;
    static_cast<AttnShape&>(a) = shape;
    a.lse = p.lse; a.delta = p.delta;
    a.dq = (uint16_t*)p.dq; a.dq_ts = p.dq_ts;
    const int max_q = p.cu_q ? (int)Tq : p.Sq;
    a.num_q_tiles = (max_q + kDqRows - 1) / kDqRows;
#define TB_DQ(DD, BF)                                                           \
  (drop ? launch_bwd_dq<DD, BF, true>(mq, mk, mv, mdo, a, stream)               \
        : launch_bwd_dq<DD, BF, false>(mq, mk, mv, mdo, a, stream))
    if (is_bf16) e = (D == 128) ? TB_DQ(128, true) : TB_DQ(64, true);
    else e = (D == 128) ? TB_DQ(128, false) : TB_DQ(64, false);
#undef TB_DQ
  }
  return e;
}

}  // namespace tb
