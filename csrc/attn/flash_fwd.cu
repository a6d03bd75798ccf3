// FlashAttention forward on wgmma / TMA for sm_90a.
//
// One CTA per (128-row query tile, q head, batch/sequence), three warpgroups:
//   warp 0     : TMA producer -- Q once, then 2-stage rings of K and V tiles (3-D tensor maps over [tokens, heads, D],
//                SWIZZLE_128B boxes of 64 x 1 x 128, so strided q/k/v views of a fused QKV activation are read in place)
//   warps 4-11 : two MMA warpgroups, 64 query rows each.  Per key tile: S = Q K^T (wgmma m64n128k16, both operands from
//                shared memory, fp32 scores in registers), scale / mask / online softmax with exp2 (a row lives in the
//                four lanes of a quad), P converted in registers to the A operand of O += P V (V read MN-major from
//                shared memory).  The two warpgroups are not synchronised with each other, so one runs its softmax
//                while the other one occupies the tensor cores.
// Masking: causal (bottom-right aligned), sliding window (left, right), per-sequence lengths (cu_seqlens) and the
// ragged tail; GQA by mapping q head h to kv head h / (Hq / Hk).
//
// Reference parity: torch_xla custom calls / flash-attn FA2 kernels used by reference torchacc/ops/flash_attn.py
// (mma.sync, sm80-class); SURVEY 2.4a rows "FA2 forward (fixed)", "FA2 varlen".
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "../common/ptx.cuh"
#include "common.cuh"
#include "mask.cuh"

namespace tb {

constexpr int kBM = 128;  // query rows per CTA
constexpr int kBN = 128;  // keys per tile
constexpr int kKVStages = 2;
constexpr int kFwdThreads = 384;  // producer warpgroup + 2 MMA warpgroups

struct FwdArgs : AttnShape {
  uint16_t* o;                 // bf16 or fp16 (kernel template)
  float* lse;
  long long o_ts;
  int num_q_tiles;
  // blockwise (ring) attention: when non-null, the epilogue merges this block into the running fp32 accumulator
  // acc [Tq, Hq, D] / lse in place (log-sum-exp merge) and writes the merged output to o; acc_init: first block
  float* acc;
  int acc_init;
};

template <int D>
struct FwdSmem {
  static constexpr int kChunks = D / 64;
  static constexpr int kQBytes = kBM * D * 2;
  static constexpr int kKBytes = kBN * D * 2;
  static constexpr int kQ = 0;
  static constexpr int kK = kQ + kQBytes;
  static constexpr int kV = kK + kKVStages * kKBytes;
  static constexpr int kBar = kV + kKVStages * kKBytes;
  static constexpr int kTotal = kBar + 256 + 1024;
};

template <int D, bool kBf16, bool kDrop>
__global__ void __launch_bounds__(kFwdThreads, 1)
flash_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const FwdArgs args) {
  using S = FwdSmem<D>;
  constexpr int kChunks = S::kChunks;

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();
  const int b = blockIdx.z, h = blockIdx.y;
  const int hk = h / (args.Hq / args.Hk);
  const int tile = args.num_q_tiles - 1 - (int)blockIdx.x;  // heavy (late) causal tiles first
  int q_start, q_len, k_start, k_len;
  seq_bounds(args, b, q_start, q_len, k_start, k_len);
  const int m0 = tile * kBM;
  if (m0 >= q_len) return;
  const bool merging = args.acc != nullptr;

  // KV tile range touched by this query tile
  int j_lo, n_tiles;
  key_tile_range(m0, kBM, q_len, k_len, args.wl, args.wr, kBN, j_lo, n_tiles);

  if (n_tiles <= 0) {  // nothing visible: O = 0, LSE = -inf (merging: the running result is unchanged)
    for (int r = threadIdx.x; r < min(kBM, q_len - m0); r += blockDim.x) {
      uint16_t* op = args.o + (long long)(q_start + m0 + r) * args.o_ts + (long long)h * D;
      if (merging && !args.acc_init) {
        const float* ap = args.acc + ((long long)(q_start + m0 + r) * args.Hq + h) * D;
        for (int d = 0; d < D; d += 2) *reinterpret_cast<uint32_t*>(op + d) = pack_h2<kBf16>(ap[d], ap[d + 1]);
        continue;
      }
      for (int d = 0; d < D; ++d) op[d] = 0;
      if (merging) {
        float* ap = args.acc + ((long long)(q_start + m0 + r) * args.Hq + h) * D;
        for (int d = 0; d < D; ++d) ap[d] = 0.f;
      }
      args.lse[(long long)h * args.Tq + q_start + m0 + r] = -INFINITY;
    }
    return;
  }

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base + S::kQ, sK = base + S::kK, sV = base + S::kV;
  const uint32_t bar = base + S::kBar;
  const uint32_t q_full = bar;
  auto k_full = [&](int s) { return bar + 8u * (1 + s); };
  auto k_empty = [&](int s) { return bar + 8u * (1 + kKVStages + s); };
  auto v_full = [&](int s) { return bar + 8u * (1 + 2 * kKVStages + s); };
  auto v_empty = [&](int s) { return bar + 8u * (1 + 3 * kKVStages + s); };

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
  }
  if (warp_idx == 1 && lane == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kKVStages; ++s) {
      mbar_init(k_full(s), 1);
      mbar_init(v_full(s), 1);
      mbar_init(k_empty(s), 2);   // one arrival per MMA warpgroup
      mbar_init(v_empty(s), 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    setmaxnreg_dec<40>();
    // ================================ TMA producer ================================
    if (warp_idx == 0 && lane == 0) {
      mbar_arrive_expect_tx(q_full, S::kQBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c) tma_load_3d(sQ + c * 16384, &tmap_q, q_full, c * 64, h, q_start + m0);
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % kKVStages;
        const uint32_t ph = ((t / kKVStages) & 1) ^ 1;
        const int tok = k_start + (j_lo + t) * kBN;
        mbar_wait(k_empty(s), ph);
        mbar_arrive_expect_tx(k_full(s), S::kKBytes);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) tma_load_3d(sK + s * S::kKBytes + c * 16384, &tmap_k, k_full(s), c * 64, hk, tok);
        mbar_wait(v_empty(s), ph);
        mbar_arrive_expect_tx(v_full(s), S::kKBytes);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) tma_load_3d(sV + s * S::kKBytes + c * 16384, &tmap_v, v_full(s), c * 64, hk, tok);
      }
    }
    return;
  }

  // ================================ MMA + softmax + epilogue ================================
  setmaxnreg_inc<232>();
  const int wg = (warp_idx >> 2) - 1;
  const uint32_t quad = lane & 3;
  const int r0 = wg * 64 + (warp_idx & 3) * 16 + (int)(lane >> 2);   // this thread's rows inside the tile: r0, r0 + 8
  const bool elected = (threadIdx.x & 127) == 0;
  int lo[2], hi[2], pos_q[2];
  uint32_t drop_row[2] = {0u, 0u};
  float lse_prev[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = min(m0 + r0 + 8 * i, q_len - 1);
    key_bounds(row, q_len, k_len, args.wl, args.wr, lo[i], hi[i]);
    pos_q[i] = row + (k_len - q_len);
    if constexpr (kDrop)
      drop_row[i] = drop_row_part(drop_head_part(args.drop.seed_lo, (uint32_t)(b * args.Hq + h)), (uint32_t)(m0 + r0 + 8 * i));
    // running LSE of the previous blocks: read before the epilogue overwrites it
    if (merging && !args.acc_init && m0 + r0 + 8 * i < q_len)
      lse_prev[i] = args.lse[(long long)h * args.Tq + q_start + m0 + r0 + 8 * i];
  }
  // ALiBi: bias -slope * |query position - key| is folded into the scores (log2 units); the softmax then runs with
  // scale 1
  const bool has_alibi = args.alibi != nullptr;
  const float slope_l2 = has_alibi ? args.alibi[(long long)b * args.alibi_bs + h] * 1.4426950408889634f : 0.f;
  const float sl2 = has_alibi ? 1.f : args.scale_log2;

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float oacc[D / 2];
  mbar_wait(q_full, 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int s = t % kKVStages;
    const uint32_t ph = (t / kKVStages) & 1;
    const int n0 = (j_lo + t) * kBN;
    // ---- S = Q K^T ----
    float sacc[kBN / 2];
    mbar_wait(k_full(s), ph);
    wgmma_fence_acc(sacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<kBN, kBf16, 0, 0>(sacc, desc_kmajor_sw128(sQ + (kk / 4) * 16384 + wg * 8192, kk % 4),
                                 desc_kmajor_sw128(sK + s * S::kKBytes + (kk / 4) * 16384, kk % 4), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sacc);
    if (elected) mbar_arrive(k_empty(s));

    // ---- scale / mask / online softmax ----
    mask_score_tile<kBN>(sacc, n0, quad, lo, hi, pos_q, has_alibi, args.scale_log2, slope_l2);
    float alpha[2], mref[2], psum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j) mx = fmaxf(mx, fmaxf(sacc[4 * j + 2 * i], sacc[4 * j + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx * sl2);
      alpha[i] = (m_run[i] == -INFINITY) ? 0.f : fast_exp2(m_run[i] - m_new);
      m_run[i] = m_new;
      mref[i] = (m_new == -INFINITY) ? 0.f : m_new;
    }
    // P = exp2(score - m) (masked entries are -inf -> 0), packed straight into the A fragments of the P V MMAs;
    // dropout masks and rescales P on its way to the MMA, the row sums use the undropped P
    uint32_t pfrag[kBN / 16][4];
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float p0 = fast_exp2(fmaf(sacc[4 * j + 2 * i], sl2, -mref[i]));
        float p1 = fast_exp2(fmaf(sacc[4 * j + 2 * i + 1], sl2, -mref[i]));
        psum[i] += p0 + p1;
        if constexpr (kDrop) {
          const uint32_t k0 = (uint32_t)(n0 + 8 * j + 2 * (int)quad);
          p0 = drop_keep(drop_row[i], drop_key_part(args.drop.seed_hi, k0), args.drop.thresh24) ? p0 * args.drop.rp : 0.f;
          p1 = drop_keep(drop_row[i], drop_key_part(args.drop.seed_hi, k0 + 1), args.drop.thresh24) ? p1 * args.drop.rp : 0.f;
        }
        pfrag[j >> 1][(j & 1) * 2 + i] = pack_h2<kBf16>(p0, p1);
      }
#pragma unroll
    for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * alpha[i] + psum[i];
    if (t > 0) {
#pragma unroll
      for (int j = 0; j < D / 8; ++j) {
        oacc[4 * j + 0] *= alpha[0]; oacc[4 * j + 1] *= alpha[0];
        oacc[4 * j + 2] *= alpha[1]; oacc[4 * j + 3] *= alpha[1];
      }
    }
    // ---- O += P V ----
    mbar_wait(v_full(s), ph);
    wgmma_fence_acc(oacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk)
      wgmma_rs<D, kBf16, 1>(oacc, pfrag[kk], desc_mnmajor_sw128(sV + s * S::kKBytes, kk, 16384), (t | kk) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(oacc);
    if (elected) mbar_arrive(v_empty(s));
  }

  // ---- epilogue: O / l -> bf16 / fp16, LSE ----
  const bool vec_o = (args.o_ts % 8 == 0) && (reinterpret_cast<uintptr_t>(args.o) % 16 == 0);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = m0 + r0 + 8 * i;
    const bool valid = row < q_len;
    const float inv_l = (l > 0.f) ? (1.f / l) : 0.f;
    const float lse_blk = (l > 0.f) ? (m_run[i] + log2f(l)) * 0.6931471805599453f : -INFINITY;
    float w_old = 0.f, w_new = inv_l, lse_out = lse_blk;
    if (merging) {
      // log-sum-exp merge with the running result: out = acc * w_old + (O / l) * w_new
      const float mx = fmaxf(lse_prev[i], lse_blk);
      w_new = 0.f;
      lse_out = -INFINITY;
      if (mx != -INFINITY) {
        const float e_old = __expf(lse_prev[i] - mx), e_new = __expf(lse_blk - mx);   // exp(-inf) == 0
        const float den = e_old + e_new;
        lse_out = mx + __logf(den);
        w_old = e_old / den;
        w_new = inv_l * e_new / den;
      }
    }
    float* ap = merging ? args.acc + ((long long)(q_start + row) * args.Hq + h) * D : nullptr;
    uint16_t* op = args.o + (long long)(q_start + row) * args.o_ts + (long long)h * D;
#pragma unroll
    for (int g = 0; g < D / 32; ++g) {
      uint32_t x[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * g + jj;
        float v0 = oacc[4 * j + 2 * i] * w_new, v1 = oacc[4 * j + 2 * i + 1] * w_new;
        if (merging && valid) {
          float2* a2 = reinterpret_cast<float2*>(ap + 8 * j + 2 * quad);
          if (!args.acc_init) {
            const float2 old = *a2;
            v0 = fmaf(old.x, w_old, v0);
            v1 = fmaf(old.y, w_old, v1);
          }
          *a2 = make_float2(v0, v1);
        }
        x[jj] = pack_h2<kBf16>(v0, v1);
      }
      quad_transpose(x, lane);
      if (valid) store_row8(op + 32 * g + 8 * quad, x, 8, vec_o);
    }
    if (valid && quad == 0) args.lse[(long long)h * args.Tq + q_start + row] = lse_out;
  }
}

template <int D, bool kBf16, bool kDrop>
static cudaError_t launch_fwd(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const FwdArgs& a,
                              cudaStream_t stream) {
  using S = FwdSmem<D>;
  auto kern = flash_fwd_kernel<D, kBf16, kDrop>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid(a.num_q_tiles, a.Hq, a.B);
  kern<<<grid, kFwdThreads, S::kTotal, stream>>>(mq, mk, mv, a);
  return cudaGetLastError();
}

cudaError_t flash_attn_fwd(const AttnParams& p, cudaStream_t stream) {
  if (p.B == 0 || p.Tq == 0) return cudaSuccess;
  FwdArgs a;
  cudaError_t e = make_shape(p, a);
  if (e != cudaSuccess) return e;
  CUtensorMap mq, mk, mv;
  try {
    mq = make_map_thd(p.q, p.Tq, p.Hq, p.D, p.q_ts, p.is_bf16, kBM);
    mk = make_map_thd(p.k, p.Tk, p.Hk, p.D, p.k_ts, p.is_bf16, kBN);
    mv = make_map_thd(p.v, p.Tk, p.Hk, p.D, p.v_ts, p.is_bf16, kBN);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  a.o = (uint16_t*)p.o;
  a.lse = p.lse;
  a.o_ts = p.o_ts;
  a.num_q_tiles = ((p.cu_q ? (int)p.Tq : p.Sq) + kBM - 1) / kBM;
  a.acc = p.acc; a.acc_init = p.acc_init;
  const bool drop = p.p_drop > 0.f;
#define TB_FWD(DD, BF) \
  (drop ? launch_fwd<DD, BF, true>(mq, mk, mv, a, stream) : launch_fwd<DD, BF, false>(mq, mk, mv, a, stream))
  if (p.is_bf16) return (p.D == 128) ? TB_FWD(128, true) : TB_FWD(64, true);
  return (p.D == 128) ? TB_FWD(128, false) : TB_FWD(64, false);
#undef TB_FWD
}

}  // namespace tb
