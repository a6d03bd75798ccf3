// Block-scaled FP8 (MX: e4m3 elements, one UE8M0 scale per 32 elements along K) GEMM on wgmma for sm_90a.
//
//   D[M,N] (bf16 or fp32, row-major) (+)= (A[M,K] * SFA) . (B[N,K] * SFB)^T        A, B: e4m3, K-major
//
// Hopper's tensor cores multiply e4m3 operands but know nothing about block scales, and one wgmma.m64n128k32 covers
// exactly one 32-element scale block.  So every K block of 32 is multiplied into a scratch accumulator and promoted into
// the fp32 result with the factor 2^(sfa-127) * 2^(sfb-127) of its (row, column) -- a power of two, so the promotion is
// exact.  Per pipeline stage (K = 128 elements = one 128-byte swizzle row):
//   warp 0     : TMA producer -- A tile 128 x 128 B, B tile 128 x 128 B (SWIZZLE_128B), plus the two scale "atoms" of the
//                stage (512 B for 128 rows x 4 K-blocks, layout written by ops/quant_mxfp8.cu) as bulk copies
//   warps 4-11 : two MMA warpgroups (64 rows each): 4 x (wgmma 64x128x32 -> scale -> accumulate), then the epilogue
//                (+ C) -> bf16/fp32 stores
// All three GEMMs of a linear layer are K-major x K-major here: the transposed operands of dgrad / wgrad come from the
// transposing quantiser (ops/quant_mxfp8.cu), because the scales must run along the contraction dimension.
//
// Grouped (mixture-of-experts) modes, selected at compile time (kGroup; 0 is the dense GEMM above), over the
// expert-sorted rows of ops/moe.py (every expert's segment padded to 128 rows, see GroupArgs in gemm_bf16.cu):
//   kGroup 1 (forward, dgrad): D[rows, N] = A[rows, K] B_e^T with e = tile_expert[m tile]; the row tiles run up to the
//     device-resident *num_m_tiles.  B_e starts b_row_step row blocks (forward: B = [E*N][K]) or b_k_step K blocks
//     (dgrad: B = the transposed quantisation [N][E*K]) after B_(e-1), in the e4m3 data and in the scale atoms alike.
//   kGroup 2 (wgrad): D[e*M + m, n] (+)= sum over r in [offsets[e], offsets[e+1]) of A[m, r] B[n, r]; tiles are
//     (expert, m, n) and the K loop covers the expert's padded rows, whole 128-row blocks, so a K block and its scale
//     atom never straddle two experts.  An expert without rows writes zeros (or leaves D unchanged when accumulating).
//
// The reference has no fp8 path at all (torchacc/config.py:27-54); BASELINE.json asks for block-scaled fp8 GEMMs.
#include <stdio.h>
#include <string.h>

#include "../common/ptx.cuh"
#include "../common/tensormap.h"
#include "gemm.h"

namespace tb {

namespace mx {

constexpr int kBM = 128, kBN = 128, kBKBytes = 128;   // tile; K block = 128 e4m3 elements
constexpr int kStages = 5;
constexpr int kThreads = 384;
constexpr int kABytes = kBM * kBKBytes;               // 16 KB
constexpr int kBBytes = kBN * kBKBytes;               // 16 KB
constexpr int kSfBytes = 512;                         // one atom: 128 rows x 4 K blocks
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSfStageBytes = 2 * kSfBytes;
constexpr int kBarBytes = 1024;
constexpr int kSmemTotal = kStages * kStageBytes + kStages * kSfStageBytes + kBarBytes + 1024;
constexpr int kGroupM = 8;

struct Args {
  void* D;
  const void* C;
  int M, N, K;
  long long ldd, ldc;
  int out_fp32;
  int num_m_tiles, num_n_tiles;
  const uint8_t* sfa;   // atom-tiled: [ceil(M/128)][K/128][512]
  const uint8_t* sfb;   // atom-tiled: [ceil(N/128)][K/128][512]
  // grouped modes only
  const int* tile_expert;    // kGroup 1: expert of every 128-row tile
  const int* m_tiles_dev;    // kGroup 1: device-resident count of valid row tiles
  const int* offsets;        // kGroup 2: [E + 1] padded row offsets, the experts' K ranges
  int num_experts;           // kGroup 2
  int sfa_katoms, sfb_katoms;   // K atoms per row block of the scale tensors
  int b_row_step, b_k_step;     // kGroup 1: B_e's first row block / K block is e times these
};

// where tile t reads and writes: row / column tile, expert, first K block of A and of B, B's row block, K blocks
struct TileRef {
  int tm, tn, e, a_k0, b_k0, b_row, nkb;
};

__device__ __forceinline__ void tile_coords(int t, int num_m_tiles, int num_n_tiles, int& tm, int& tn) {
  const int per_group = kGroupM * num_n_tiles;
  const int g = t / per_group;
  const int first_m = g * kGroupM;
  const int gsize = min(kGroupM, num_m_tiles - first_m);
  const int r = t - g * per_group;
  tm = first_m + (r % gsize);
  tn = r / gsize;
}

// the four UE8M0 scales (K blocks 0-3 of the stage) of row r of a 128-row atom
TB_DEVICE uint32_t ld_sf4(uint32_t atom, int r) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(atom + (uint32_t)((r & 31) * 16 + (r >> 5) * 4)));
  return v;
}
TB_DEVICE float sf_value(uint32_t sf4, int kq) {   // 2^(e-127); e == 0 is the subnormal 2^-127
  const uint32_t e = (sf4 >> (8 * kq)) & 0xffu;
  return __uint_as_float(e != 0 ? e << 23 : 0x00400000u);
}

template <int kGroup>
__device__ __forceinline__ TileRef locate(int t, const Args& args, int num_m_tiles, int num_k_blocks) {
  TileRef p;
  int u = t;
  p.e = 0;
  if constexpr (kGroup == 2) {
    p.e = t / (num_m_tiles * args.num_n_tiles);
    u = t - p.e * (num_m_tiles * args.num_n_tiles);
  }
  tile_coords(u, num_m_tiles, args.num_n_tiles, p.tm, p.tn);
  p.a_k0 = 0;
  p.b_k0 = 0;
  p.b_row = p.tn;
  p.nkb = num_k_blocks;
  if constexpr (kGroup == 1) {
    p.e = args.tile_expert[p.tm];
    p.b_row += p.e * args.b_row_step;
    p.b_k0 = p.e * args.b_k_step;
  } else if constexpr (kGroup == 2) {
    p.a_k0 = p.b_k0 = args.offsets[p.e] / kBKBytes;
    p.nkb = args.offsets[p.e + 1] / kBKBytes - p.a_k0;
  }
  return p;
}

template <int kGroup>
__global__ void __launch_bounds__(kThreads, 1)
gemm_mxfp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const Args args) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sf_base = smem_base + kStages * kStageBytes;
  const uint32_t bar_base = sf_base + kStages * kSfStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  auto smem_a = [&](int s) { return smem_base + s * kStageBytes; };
  auto smem_b = [&](int s) { return smem_base + s * kStageBytes + kABytes; };
  auto smem_sfa = [&](int s) { return sf_base + s * kSfStageBytes; };
  auto smem_sfb = [&](int s) { return sf_base + s * kSfStageBytes + kSfBytes; };

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();
  int num_m_tiles = args.num_m_tiles;
  if constexpr (kGroup == 1) num_m_tiles = *args.m_tiles_dev;
  const int num_tiles = num_m_tiles * args.num_n_tiles * (kGroup == 2 ? args.num_experts : 1);
  const int num_k_blocks = args.K / kBKBytes;
  // the dense GEMM's scale tensors have exactly K / 128 atoms per row block
  const int sfa_katoms = kGroup == 0 ? num_k_blocks : args.sfa_katoms;
  const int sfb_katoms = kGroup == 0 ? num_k_blocks : args.sfb_katoms;

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
  }
  if (warp_idx == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    setmaxnreg_dec<40>();
    // ================================ TMA producer ================================
    if (warp_idx == 0 && lane == 0) {
      int it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileRef p = locate<kGroup>(t, args, num_m_tiles, num_k_blocks);
        for (int kb = 0; kb < p.nkb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(empty_bar(s), ((it / kStages) & 1) ^ 1);
          mbar_arrive_expect_tx(full_bar(s), kStageBytes + kSfStageBytes);
          tma_load_2d(smem_a(s), &tmap_a, full_bar(s), (p.a_k0 + kb) * kBKBytes, p.tm * kBM);
          tma_load_2d(smem_b(s), &tmap_b, full_bar(s), (p.b_k0 + kb) * kBKBytes, p.b_row * kBN);
          bulk_load(smem_sfa(s), args.sfa + ((size_t)p.tm * sfa_katoms + p.a_k0 + kb) * 512, kSfBytes, full_bar(s));
          bulk_load(smem_sfb(s), args.sfb + ((size_t)p.b_row * sfb_katoms + p.b_k0 + kb) * 512, kSfBytes, full_bar(s));
        }
      }
    }
    return;
  }

  // ================================ MMA + promotion + epilogue ================================
  setmaxnreg_inc<232>();
  const int wg = (warp_idx >> 2) - 1;
  const uint32_t quad = lane & 3;
  const int frag_row = wg * 64 + (warp_idx & 3) * 16 + (int)(lane >> 2);   // rows frag_row, frag_row + 8 of the tile
  int it = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const TileRef p = locate<kGroup>(t, args, num_m_tiles, num_k_blocks);
    const int tm = p.tm, tn = p.tn;
    float acc[kBN / 2];
#pragma unroll
    for (int i = 0; i < kBN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < p.nkb; ++kb, ++it) {
      const int s = it % kStages;
      mbar_wait(full_bar(s), (it / kStages) & 1);
      const uint32_t sa4[2] = {ld_sf4(smem_sfa(s), frag_row), ld_sf4(smem_sfa(s), frag_row + 8)};
#pragma unroll
      for (int kq = 0; kq < 4; ++kq) {
        float part[kBN / 2];
        wgmma_fence_acc(part);
        wgmma_fence();
        wgmma_ss_e4m3_n128(part, desc_kmajor_sw128(smem_a(s) + wg * 8192, kq), desc_kmajor_sw128(smem_b(s), kq), 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(part);
        const float sa0 = sf_value(sa4[0], kq), sa1 = sf_value(sa4[1], kq);
#pragma unroll
        for (int j = 0; j < kBN / 8; ++j) {
          const int c = 8 * j + 2 * (int)quad;
          const float sb0 = sf_value(ld_sf4(smem_sfb(s), c), kq), sb1 = sf_value(ld_sf4(smem_sfb(s), c + 1), kq);
          acc[4 * j + 0] = fmaf(part[4 * j + 0], sa0 * sb0, acc[4 * j + 0]);
          acc[4 * j + 1] = fmaf(part[4 * j + 1], sa0 * sb1, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(part[4 * j + 2], sa1 * sb0, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(part[4 * j + 3], sa1 * sb1, acc[4 * j + 3]);
        }
      }
      __syncwarp();
      // every thread of the group has finished reading the stage (its MMAs retired and its scales are in registers)
      if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory"); else asm volatile("bar.sync 2, 128;" ::: "memory");
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar(s));
    }

    const long long row0 = (long long)tm * kBM + frag_row;
    const int n0 = tn * kBN;
    // wgrad: expert e owns rows [e * M, e * M + M) of D (and of C)
    const long long erow = kGroup == 2 ? (long long)p.e * args.M : 0;
    if (args.out_fp32) {
      const bool vec = (args.ldd % 2 == 0) && (args.C == nullptr || args.ldc % 2 == 0) &&
                       (reinterpret_cast<uintptr_t>(args.D) % 8 == 0) && (reinterpret_cast<uintptr_t>(args.C) % 8 == 0);
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * (int)quad;
        if (col >= args.N) continue;
        const bool two = col + 1 < args.N;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const long long grow = row0 + 8 * half;
          if (grow >= args.M) continue;
          float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
          float* dp = reinterpret_cast<float*>(args.D) + (erow + grow) * args.ldd + col;
          const float* cp = args.C ? reinterpret_cast<const float*>(args.C) + (erow + grow) * args.ldc + col : nullptr;
          if (two && vec) {
            if (cp) {
              const float2 old = *reinterpret_cast<const float2*>(cp);
              v0 += old.x; v1 += old.y;
            }
            *reinterpret_cast<float2*>(dp) = make_float2(v0, v1);
          } else {
            dp[0] = v0 + (cp ? cp[0] : 0.f);
            if (two) dp[1] = v1 + (cp ? cp[1] : 0.f);
          }
        }
      }
    } else {
      const bool vec_d = (args.ldd % 8 == 0) && (reinterpret_cast<uintptr_t>(args.D) % 16 == 0);
#pragma unroll
      for (int g = 0; g < kBN / 32; ++g) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const long long grow = row0 + 8 * half;
          const bool row_ok = grow < args.M;
          uint32_t x[4];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * g + jj;
            const int col = n0 + 8 * j + 2 * (int)quad;
            float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
            if (args.C != nullptr && row_ok && col < args.N) {
              const __nv_bfloat16* cp = reinterpret_cast<const __nv_bfloat16*>(args.C) + (erow + grow) * args.ldc + col;
              v0 += __bfloat162float(cp[0]);
              if (col + 1 < args.N) v1 += __bfloat162float(cp[1]);
            }
            x[jj] = pack_bf16x2(v0, v1);
          }
          quad_transpose(x, lane);
          const int col = n0 + 32 * g + 8 * (int)quad;
          if (row_ok && col < args.N)
            store_row8(reinterpret_cast<uint16_t*>(args.D) + (erow + grow) * args.ldd + col, x, args.N - col, vec_d);
        }
      }
    }
  }
}

}  // namespace mx

static CUtensorMap make_map_2d_u8(const void* base, uint64_t rows, uint64_t cols, uint64_t ld_bytes, uint32_t box_cols,
                                  uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld_bytes};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tensor_map(base, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int kGroup>
static cudaError_t launch_mxfp8(const CUtensorMap& ta, const CUtensorMap& tbm, const mx::Args& a, int num_tiles,
                                int num_sms, cudaStream_t stream) {
  static cudaError_t cfg = cudaFuncSetAttribute(mx::gemm_mxfp8_kernel<kGroup>,
                                                cudaFuncAttributeMaxDynamicSharedMemorySize, mx::kSmemTotal);
  if (cfg != cudaSuccess) return cfg;
  int grid = num_tiles;
  if (grid > num_sms) grid = num_sms;
  mx::gemm_mxfp8_kernel<kGroup><<<grid, mx::kThreads, mx::kSmemTotal, stream>>>(ta, tbm, a);
  return cudaGetLastError();
}

static mx::Args mx_args(const void* sfa, const void* sfb, void* D, const void* C, int M, int N, int K, long long ldd,
                        long long ldc, bool out_fp32) {
  mx::Args a;
  memset(&a, 0, sizeof(a));
  a.D = D; a.C = C; a.M = M; a.N = N; a.K = K; a.ldd = ldd; a.ldc = ldc; a.out_fp32 = out_fp32 ? 1 : 0;
  a.num_m_tiles = (M + mx::kBM - 1) / mx::kBM;
  a.num_n_tiles = (N + mx::kBN - 1) / mx::kBN;
  a.sfa = reinterpret_cast<const uint8_t*>(sfa);
  a.sfb = reinterpret_cast<const uint8_t*>(sfb);
  return a;
}

// A: [M][K] e4m3 (row pitch lda bytes), B: [N][K] e4m3; sfa / sfb: atom-tiled UE8M0 scales (see quant_mxfp8.cu).
cudaError_t gemm_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, const void* C, int M,
                       int N, int K, long long lda, long long ldb, long long ldd, long long ldc, bool out_fp32,
                       int num_sms, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K <= 0 || K % 128 != 0 || lda % 16 != 0 || ldb % 16 != 0) return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_u8(A, M, K, lda, mx::kBKBytes, mx::kBM);
    tbm = make_map_2d_u8(B, N, K, ldb, mx::kBKBytes, mx::kBN);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  const mx::Args a = mx_args(sfa, sfb, D, C, M, N, K, ldd, ldc, out_fp32);
  return launch_mxfp8<0>(ta, tbm, a, a.num_m_tiles * a.num_n_tiles, num_sms, stream);
}

// Grouped forward / dgrad over expert-sorted rows (kGroup 1).  A: [M][K] e4m3, M the padded row capacity.
//   b_transposed == false (forward): B = [E*N][K], scales [E*N/128][K/128] atoms; N % 128 == 0.
//   b_transposed == true  (dgrad):   B = [N][E*K] (transposed quantisation of the [E*K][N] weight), scales
//                                    [ceil(N/128)][E*K/128] atoms.
cudaError_t gemm_grouped_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, int M, int N,
                               int K, int E, long long lda, long long ldb, long long ldd, bool b_transposed,
                               const int* tile_expert, const int* num_m_tiles, int num_sms, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K <= 0 || K % 128 != 0 || E <= 0 || M % mx::kBM != 0 || lda % 16 != 0 || ldb % 16 != 0)
    return cudaErrorInvalidValue;
  if ((!b_transposed && N % mx::kBN != 0) || tile_expert == nullptr || num_m_tiles == nullptr)
    return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_u8(A, M, K, lda, mx::kBKBytes, mx::kBM);
    tbm = b_transposed ? make_map_2d_u8(B, N, (uint64_t)E * K, ldb, mx::kBKBytes, mx::kBN)
                       : make_map_2d_u8(B, (uint64_t)E * N, K, ldb, mx::kBKBytes, mx::kBN);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  mx::Args a = mx_args(sfa, sfb, D, nullptr, M, N, K, ldd, 0, false);
  a.tile_expert = tile_expert;
  a.m_tiles_dev = num_m_tiles;
  a.sfa_katoms = K / 128;
  a.sfb_katoms = b_transposed ? E * (K / 128) : K / 128;
  a.b_row_step = b_transposed ? 0 : N / mx::kBN;
  a.b_k_step = b_transposed ? K / 128 : 0;
  // the grid is sized by the capacity; the kernel reads the real row tile count on the device
  return launch_mxfp8<1>(ta, tbm, a, a.num_m_tiles * a.num_n_tiles, num_sms, stream);
}

// Grouped wgrad (kGroup 2): D[e*M + m, n] (+)= sum over expert e's padded rows r of A[m, r] B[n, r].  A = [M][rows],
// B = [N][rows]: the transposed quantisations of dY and X, scales along the rows ([ceil(M/128)][rows/128] atoms).
cudaError_t gemm_grouped_wgrad_mxfp8(const void* A, const void* sfa, const void* B, const void* sfb, void* D, int M,
                                     int N, int E, int rows, long long lda, long long ldb, long long ldd,
                                     const int* offsets, bool out_fp32, bool accumulate, int num_sms,
                                     cudaStream_t stream) {
  if (M <= 0 || N <= 0 || E <= 0) return cudaSuccess;
  if (rows <= 0 || rows % 128 != 0 || lda % 16 != 0 || ldb % 16 != 0 || offsets == nullptr)
    return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_u8(A, M, rows, lda, mx::kBKBytes, mx::kBM);
    tbm = make_map_2d_u8(B, N, rows, ldb, mx::kBKBytes, mx::kBN);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  mx::Args a = mx_args(sfa, sfb, D, accumulate ? D : nullptr, M, N, rows, ldd, ldd, out_fp32);
  a.offsets = offsets;
  a.num_experts = E;
  a.sfa_katoms = a.sfb_katoms = rows / 128;
  return launch_mxfp8<2>(ta, tbm, a, E * a.num_m_tiles * a.num_n_tiles, num_sms, stream);
}

}  // namespace tb
