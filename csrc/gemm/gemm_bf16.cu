// Persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] (row-major) (+)= A_op[M,K] * B_op[N,K]^T (+ bias[N])
//
// Each operand may be stored K-major (reduction dim contiguous) or MN-major (M / N contiguous), so the
// one kernel covers the three GEMMs of a linear layer without any transposes in memory:
//   forward  y  = x  W^T : A = x  (K-major),  B = W  (K-major)
//   dgrad    dx = dy W   : A = dy (K-major),  B = W  (MN-major)
//   wgrad    dW = dy^T x : A = dy (MN-major), B = x  (MN-major)
//
// Structure (one CTA of three warpgroups per SM, 128 x 256 output tile):
//   warp 0     : TMA producer   (cp.async.bulk.tensor -> 128B-swizzled smem ring of 4 stages, mbarrier full/empty)
//   warp 3     : carried collective (slices of pending FSDP transfers, fused/carry.cuh)
//   warps 4-11 : two MMA warpgroups, 64 rows each: wgmma.mma_async m64n256k16 with both operands read from shared
//                memory, fp32 accumulators in registers (128 per thread; the producer warpgroup hands its registers
//                over with setmaxnreg), then the epilogue (bias / addend / cast, 16-byte stores after a quad transpose)
// While the MMA warpgroups run the epilogue of tile i, the producer already fills the ring with tile i+1.
// Dense launches with aligned outputs and nothing to carry stage the epilogue instead (kStaged): fragments go to
// 128B-swizzled shared-memory boxes that one thread per warpgroup stores (or reduce-adds) with TMA, and a 16-bit
// addend arrives in those boxes by TMA, so the MMA warpgroups never wait on global memory between two tiles.
// Dense launches with nothing to carry run an instantiation without warp 3's role (kCarry == false): the role's
// function calls (printf, 64-bit division) make ptxas serialise every wgmma of a kernel (warning C7510), so that each
// m64n256k16 waits for the previous one.  Without them the four wgmmas of a K block are in flight together.
//
// Reference parity: replaces the cuBLAS GEMMs the reference reaches through nn.Linear
// (reference torchacc/__init__.py:97-98 forces XLA onto cuBLAS; eager path uses cuBLASLt).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../common/ptx.cuh"
#include "../common/tensormap.h"
#include "../fused/carry.cuh"
#include "../fused/carry.h"
#include "gemm.h"

namespace tb {

constexpr int kBlockM = 128;     // accumulator rows per CTA (64 per MMA warpgroup)
constexpr int kBlockN = 256;     // wgmma N
constexpr int kBlockK = 64;      // 128 bytes of bf16 = one swizzle row
constexpr int kNumThreads = 384;
constexpr int kCommCtasPerCluster = 2;   // the fused all-gather counts its copy engines in pairs of CTAs
enum class Major { K, MN };
constexpr int kGroupM = 8;       // tile rasterisation: sweep 8 row-tiles before moving along N

constexpr int kMaxPeers = 8;

// Fusion of the GEMM with the adjacent tensor-parallel collective over NVLink peer memory.
//   kFuse == 1 (all-gather -> GEMM): the A operand is the token-gathered activation.  Every rank owns a symmetric
//     [world*rows, K] buffer and has already written ITS row block; the leading 2 * `comm_clusters` CTAs of this
//     kernel pull the other ranks' row blocks from peer memory into the local buffer and publish one ready counter
//     per source rank; the GEMM CTAs consume M-tiles in shard order (own block first) and their TMA producers
//     spin on the counter of the shard they are about to read.  The transfer of shard r+1 overlaps the MMAs of shard r.
//   kFuse == 2 (GEMM -> reduce-scatter): output row block d belongs to rank d.  The epilogue stores the bf16 partial
//     tile straight into rank d's staging slot [my_rank] with peer stores and bumps a per-(dst, src) arrival counter
//     (release.sys); a small reduce kernel on each rank sums the `world` slots in fp32 once all sources have arrived.
struct FuseArgs {
  void* peer[kMaxPeers];          // kFuse 1: peers' gathered-A buffers; kFuse 2: peers' staging buffers
  uint32_t* pads[kMaxPeers];      // symmetric signal pads (entry / exit barriers)
  uint32_t* peer_cnt[kMaxPeers];  // kFuse 2: peers' arrival counters (array of `world` uint32 per rank)
  void* a_full;                   // kFuse 1: local gathered buffer
  uint32_t* flags;                // kFuse 1: local per-source ready counters
  uint32_t* block_counter;        // exit barrier bookkeeping (local)
  int rank, world, rows_per_rank, channel;
  uint32_t epoch;                 // monotonically increasing per call on this channel
  uint32_t flag_target;           // kFuse 1: counter value that means "shard complete" for this call
  int comm_clusters;              // kFuse 1: pairs of leading CTAs acting as copy engines
  long long slot_stride;          // kFuse 2: elements between two source slots of a staging buffer
};

// Grouped (mixture-of-experts) mode, a compile-time switch of the kernel (kGroup; 0 = the dense GEMM).  The A rows
// are tokens sorted by expert, each expert's segment padded with zero rows to a multiple of kBlockM, so that no
// 128-row tile and no 64-row K block straddles two experts.  Expert weights are one flat 2-D tensor.
//   kGroup == 1 (forward, dgrad, SwiGLU gate|up):  D[Mp, N] = A[Mp, K] B_e^T with e = tile_expert[m_tile].
//     B is [E * b_rows, K] (K-major: expert e starts at row e * b_rows) or [E * b_rows, N] (MN-major: the K coordinate
//     moves by e * b_rows).  The grid covers the upper bound of row tiles; the real count lives on the device and
//     tiles past it exit at once.
//   kGroup == 2 (wgrad):  D_e[M, N] = A_e^T B_e for every expert, A = dY [Mp, M] and B = X [Mp, N] both MN-major,
//     the reduction running over the expert's padded row range [offsets[e], offsets[e+1]).  D is [E * M, N].
//     An expert without rows writes zeros (or leaves D unchanged when accumulating).
struct GroupArgs {
  const int* tile_expert;  // kGroup 1
  const int* num_m_tiles;  // kGroup 1: device-resident count of valid row tiles
  const int* offsets;      // kGroup 2: [E + 1] padded row offsets
  int num_experts;         // kGroup 2
  int b_rows;              // kGroup 1: rows of one expert in the flat B
};

struct GemmArgs {
  void* D;
  const __nv_bfloat16* bias;
  int M, N, K;
  long long ldd;
  const void* C;   // optional addend with D's dtype: D = result (+ bias) + C.  C == D is gradient accumulation;
  long long ldc;   // a different C fuses a residual add into the epilogue (h + x W^T).
  int out_fp32;
  int num_m_tiles, num_n_tiles;
  // SwiGLU epilogue (gate|up projection): B is W_gu [2F][K]; a stage holds 128 gate rows followed by the matching 128
  // up rows, so accumulator columns [0,128) / [128,256) are gate / up of the SAME 128 output columns and the
  // epilogue writes h = silu(g) * u [M][F] directly (and g|u [M][2F] only when the backward needs it).
  int swiglu;      // 0 / 1
  int swiglu_F;    // F = intermediate size
  void* gu_out;    // optional [M][2F] pre-activation (nullptr: not materialised)
  long long ldgu;
  int dynamic;     // 1: grid = one CTA per tile instead of a persistent grid (see gemm_sched_mode)
  FuseArgs fuse;
  CarryArgs carry;  // slices of pending FSDP collectives moved by warp 3 of every CTA while the tiles run (fused/carry.cuh)
  GroupArgs group;
};

TB_DEVICE void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
TB_DEVICE uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
TB_DEVICE uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
TB_DEVICE void red_release_sys_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
TB_DEVICE void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
TB_DEVICE uint4 ld_volatile_v4(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// Cross-rank barrier on the symmetric signal pad (slot layout as in comm/symm_comm.cu: 16 words per channel,
// [0,8) entry flags, [8,16) exit flags).  `signal` is true for exactly one CTA per rank.
// `tid` enumerates the calling threads (threadIdx.x for a whole CTA, the lane id for a single warp).
TB_DEVICE void fused_barrier(const FuseArgs& f, bool signal, int slot_base, int tid) {
  if (signal && tid < f.world) {
    __threadfence_system();
    st_release_sys_u32(f.pads[tid] + f.channel * 16 + slot_base + f.rank, f.epoch);
  }
  if (tid < f.world)
    spin_until_epoch(f.pads[f.rank] + f.channel * 16 + slot_base + tid, f.epoch, f.rank, tid, f.channel,
                     "fused GEMM barrier");
}

// Copy-engine role of the all-gather -> GEMM kernel (executed by whole CTAs).  One thread per CTA drives a ring
// of 32 KB TMA bulk copies  peer HBM --NVLink--> smem --> local gathered buffer:  (stages-1) x 32 KB are in flight per
// CTA, so a handful of CTAs keep the link full (16-byte register loads would need ~100 CTAs for the same bytes in
// flight).  Shard r is announced to the GEMM CTAs' TMA producers through flags[r] when all copy CTAs finished it.
TB_DEVICE void gather_role(const FuseArgs& f, int K, int comm_cta, int num_comm_ctas, uint32_t smem_base,
                           uint32_t bar_base, int num_stages) {
  constexpr uint32_t kChunk = 32768;
  if (threadIdx.x == 0) {
    for (int s = 0; s < num_stages; ++s) mbar_init(bar_base + 8u * s, 1);
    fence_mbar_init();
  }
  fused_barrier(f, comm_cta == 0, 0, threadIdx.x);   // every rank has written its own row block
  __syncthreads();
  if (threadIdx.x == 0 && f.world > 1) {
    const size_t shard_bytes = (size_t)f.rows_per_rank * K * 2;
    const int chunks = (int)(shard_bytes / kChunk);            // rows % 256 == 0 and K % 64 == 0 -> exact
    const int per = chunks > comm_cta ? (chunks - comm_cta + num_comm_ctas - 1) / num_comm_ctas : 0;
    const int total = per * (f.world - 1);
    auto locate = [&](int j, const uint8_t*& src, uint8_t*& dst) {
      const int r = (f.rank + 1 + j / per) % f.world;
      const size_t off = (size_t)r * shard_bytes + (size_t)(comm_cta + (j % per) * num_comm_ctas) * kChunk;
      src = reinterpret_cast<const uint8_t*>(f.peer[r]) + off;
      dst = reinterpret_cast<uint8_t*>(f.a_full) + off;
    };
    auto issue = [&](int j) {
      const uint8_t* src; uint8_t* dst;
      locate(j, src, dst);
      const int s = j % num_stages;
      mbar_arrive_expect_tx(bar_base + 8u * s, kChunk);
      bulk_load(smem_base + s * kChunk, src, kChunk, bar_base + 8u * s);
    };
    int issued = 0;
    for (; issued < num_stages - 1 && issued < total; ++issued) issue(issued);
    for (int i = 0; i < total; ++i) {
      const int s = i % num_stages;
      mbar_wait(bar_base + 8u * s, (i / num_stages) & 1);
      const uint8_t* src; uint8_t* dst;
      locate(i, src, dst);
      bulk_store(dst, smem_base + s * kChunk, kChunk);
      tma_store_commit();
      if (issued < total) {
        tma_store_wait_read<1>();       // every store but the newest has left smem -> stage (i-1) % stages is free
        issue(issued++);
      }
      if ((i + 1) % per == 0) {         // last chunk of a source rank handled by this CTA
        tma_store_wait<0>();            // writes complete
        __threadfence();
        atomicAdd(f.flags + (f.rank + 1 + i / per) % f.world, 1u);
      }
    }
    if (per == 0)                       // more copy CTAs than chunks: still count towards every shard's flag
      for (int st = 1; st < f.world; ++st) atomicAdd(f.flags + (f.rank + st) % f.world, 1u);
  }
  // exit: all my copy CTAs are done reading peers -> tell them; stay until every peer is done reading me
  __shared__ uint32_t s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = (atomicAdd(f.block_counter, 1u) == (uint32_t)num_comm_ctas - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) *f.block_counter = 0;
  fused_barrier(f, true, 8, threadIdx.x);
}

struct GemmSmem {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = kBlockN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = 4;
  static constexpr int kBarrierBytes = 1024;
  static constexpr int kTotal = kStages * kStageBytes + kBarrierBytes + 1024;  // +1024 alignment slack
  static constexpr int kTotalCarry = kTotal + kCarrySmemBytes;                 // + the copy warp's private ring
  // staged epilogue: two 8 KB buffers per MMA warpgroup, each one 128B-swizzled TMA box of 64 rows x 128 bytes
  static constexpr int kStagingBytes = 2 * 2 * 8192;
  static constexpr int kTotalStaged = kTotal + kStagingBytes;
  static_assert(kTotalStaged <= 227 * 1024, "staging does not fit next to the ring");
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

// tile order for the fused variants: row blocks ("shards") are visited in ring order starting from `first`
__device__ __forceinline__ void tile_coords_sharded(int t, int tiles_m_per_shard, int num_n_tiles, int first, int world,
                                                    int& tm, int& tn, int& shard) {
  const int per_shard = tiles_m_per_shard * num_n_tiles;
  const int si = t / per_shard;
  shard = (first + si) % world;
  int lm, ln;
  tile_coords(t - si * per_shard, tiles_m_per_shard, num_n_tiles, lm, ln);
  tm = shard * tiles_m_per_shard + lm;
  tn = ln;
}

// Tensor maps of the staged epilogue (kStaged): D (16-bit: 64 x 64 boxes, fp32: 32 x 64), the 16-bit addend C, and
// the SwiGLU pre-activation g|u.  Unused maps are left zeroed.
struct EpiMaps {
  CUtensorMap d, c, gu;
};

template <bool kBf16, Major kAMajor, Major kBMajor, int kFuse, int kGroup = 0, bool kCarry = true, bool kStaged = false>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmArgs args, const __grid_constant__ EpiMaps maps) {
  using S = GemmSmem;
  constexpr int kStages = S::kStages;
  constexpr int kTA = (kAMajor == Major::MN) ? 1 : 0, kTB = (kBMajor == Major::MN) ? 1 : 0;
  static_assert(kGroup == 0 || kFuse == 0, "grouped GEMMs are not fused with collectives");
  static_assert(!kStaged || (kFuse == 0 && kGroup == 0 && !kCarry), "the staged epilogue is for plain dense launches");
  static_assert(kGroup != 2 || (kAMajor == Major::MN && kBMajor == Major::MN), "grouped wgrad reads both operands MN-major");

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + kStages * S::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  auto smem_a = [&](int s) { return smem_base + s * S::kStageBytes; };
  auto smem_b = [&](int s) { return smem_base + s * S::kStageBytes + S::kABytes; };

  const int warp_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const uint32_t lane = lane_id();

  int num_m_tiles = args.num_m_tiles;
  if constexpr (kGroup == 1) num_m_tiles = *args.group.num_m_tiles;
  const int tiles_per_expert = num_m_tiles * args.num_n_tiles;
  const int num_tiles = (kGroup == 2) ? args.group.num_experts * tiles_per_expert : tiles_per_expert;
  const int num_k_blocks = (args.K + kBlockK - 1) / kBlockK;
  // grouped wgrad: the K loop covers the padded rows of expert e (multiples of kBlockM, so whole K blocks)
  auto expert_k_blocks = [&](int e, int& k_base) {
    k_base = args.group.offsets[e];
    return (args.group.offsets[e + 1] - k_base) / kBlockK;
  };
  int cta = blockIdx.x;
  int num_ctas = gridDim.x;
  if constexpr (kFuse == 1) {
    const int cc = args.fuse.comm_clusters * kCommCtasPerCluster;
    if (cta < cc) {   // copy-engine CTAs: no MMA
      gather_role(args.fuse, args.K, cta, cc, smem_base, bar_base, kStages * S::kStageBytes / 32768);
      return;
    }
    cta -= cc;
    num_ctas -= cc;
  }
  const int tiles_m_per_shard = (kFuse != 0) ? args.fuse.rows_per_rank / kBlockM : 0;
  // fused tile order: all-gather starts with the local row block; reduce-scatter ends with it (peers first)
  const int first_shard = (kFuse == 1) ? args.fuse.rank : ((kFuse == 2) ? (args.fuse.rank + 1) % args.fuse.world : 0);
  // `shard`: the row block of the fused variants, the expert of the grouped wgrad, 0 otherwise
  auto coords = [&](int t, int& tm, int& tn, int& shard) {
    if constexpr (kFuse != 0) {
      tile_coords_sharded(t, tiles_m_per_shard, args.num_n_tiles, first_shard, args.fuse.world, tm, tn, shard);
    } else if constexpr (kGroup == 2) {
      shard = t / tiles_per_expert;
      tile_coords(t - shard * tiles_per_expert, num_m_tiles, args.num_n_tiles, tm, tn);
    } else {
      shard = 0;
      tile_coords(t, num_m_tiles, args.num_n_tiles, tm, tn);
    }
  };

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (kStaged) {
      tma_prefetch_desc(&maps.d);
      if (args.C != nullptr && !args.out_fp32) tma_prefetch_desc(&maps.c);
      if (args.gu_out != nullptr) tma_prefetch_desc(&maps.gu);
    }
  }
  if (warp_idx == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per MMA warpgroup
    }
    if constexpr (kStaged) {
      for (int b = 0; b < 4; ++b) mbar_init(bar_base + 8u * (2 * kStages + b), 1);   // addend loads, see below
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    // the producer warpgroup gives its registers to the two MMA warpgroups (128 accumulator registers per thread)
    setmaxnreg_dec<56>();
    if (warp_idx == 0) {
      // ================================ TMA producer ================================
      if (lane == 0) {
        int it = 0;
        for (int t = cta; t < num_tiles; t += num_ctas) {
          int tm, tn, shard;
          coords(t, tm, tn, shard);
          const int m0 = tm * kBlockM;
          // SwiGLU: accumulator columns [0,128) are gate rows, [128,256) the matching up rows of W_gu
          const int n0 = (kFuse == 0 && args.swiglu) ? tn * (kBlockN / 2) : tn * kBlockN;
          const int n1 = (kFuse == 0 && args.swiglu) ? args.swiglu_F + n0 : n0 + kBlockN / 2;
          if constexpr (kFuse == 1) {
            if (shard != args.fuse.rank) {   // wait until the copy CTAs have landed this source rank's rows
              spin_until_count(args.fuse.flags + shard, args.fuse.flag_target, args.fuse.rank, shard,
                               "all-gather -> GEMM shard flag");
              fence_proxy_async_all();       // generic-proxy writes of the copy CTAs -> visible to TMA
            }
          }
          int nkb = num_k_blocks, k_base = 0, b_off = 0;   // b_off: the expert's offset in the flat B
          if constexpr (kGroup == 1) b_off = args.group.tile_expert[tm] * args.group.b_rows;
          if constexpr (kGroup == 2) nkb = expert_k_blocks(shard, k_base);
          for (int kb = 0; kb < nkb; ++kb, ++it) {
            const int s = it % kStages;
            mbar_wait(empty_bar(s), ((it / kStages) & 1) ^ 1);
            mbar_arrive_expect_tx(full_bar(s), S::kStageBytes);
            const int k0 = k_base + kb * kBlockK;
            if constexpr (kAMajor == Major::K) {
              tma_load_2d(smem_a(s), &tmap_a, full_bar(s), k0, m0);
            } else {
#pragma unroll
              for (int i = 0; i < kBlockM / 64; ++i)
                tma_load_2d(smem_a(s) + i * 8192, &tmap_a, full_bar(s), m0 + i * 64, k0);
            }
            if constexpr (kBMajor == Major::K) {
              tma_load_2d(smem_b(s), &tmap_b, full_bar(s), k0, b_off + n0);
              tma_load_2d(smem_b(s) + S::kBBytes / 2, &tmap_b, full_bar(s), k0, b_off + n1);
            } else {
#pragma unroll
              for (int i = 0; i < kBlockN / 64; ++i)
                tma_load_2d(smem_b(s) + i * 8192, &tmap_b, full_bar(s), n0 + i * 64, b_off + k0);
            }
          }
        }
      }
    } else if (warp_idx == 3) {
      // ================================ Carried collective ================================
      // Under static scheduling this warp moves this launch's slice of the pending FSDP all-gather / reduce-scatter
      // (TMA bulk copies through a private 24 KB ring) while the tiles are computed.  Compiled only into the
      // instantiations that launches with something to carry use (see kCarry in the header comment).
      if constexpr (kFuse == 0 && kCarry) {
        if (!args.dynamic && args.carry.slice[0].kind != 0) {
          const uint32_t ring = bar_base + S::kBarrierBytes;
          carry_role(args.carry, ring, ring + kCarryStages * kCarryStageBytes, (int)blockIdx.x, (int)gridDim.x);
        }
      }
    }
  } else {
    // ================================ MMA + epilogue (two warpgroups, 64 rows each) ================================
    setmaxnreg_inc<224>();
    const int wg = (warp_idx >> 2) - 1;              // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp_idx & 3;
    const uint32_t quad = lane & 3;
    const int frag_row = wg * 64 + wq * 16 + (int)(lane >> 2);
    auto pk = [&](float a, float b) { return pack_h2<kBf16>(a, b); };
    auto ld1 = [&](const uint16_t* p) {
      return kBf16 ? __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p))
                   : __half2float(*reinterpret_cast<const __half*>(p));
    };
    if constexpr (kFuse == 2) {
      // nobody may write into a peer's staging buffer before that peer finished reducing the previous call
      fused_barrier(args.fuse, blockIdx.x == 0 && warp_idx == 4, 0, (int)lane);
      __syncwarp();
    }
    // kFuse == 2: arrivals are batched per destination rank -- ONE system-scope fence + counter add per warp and
    // shard instead of one per tile (a fence.sys costs an NVLink round trip, longer than a whole K=2048 mainloop).
    int cur_shard = -1;
    uint32_t pending = 0;
    auto flush_arrivals = [&]() {
      if constexpr (kFuse == 2) {
        if (pending != 0) {
          __threadfence_system();
          __syncwarp();
          if (lane == 0) red_release_sys_add(args.fuse.peer_cnt[cur_shard] + args.fuse.rank, pending);
          pending = 0;
        }
      }
    };
    // Staged epilogue (kStaged): each warpgroup writes its 64 rows chunk by chunk into one of its two 8 KB staging
    // buffers (128B-swizzled, one TMA box each), and one elected thread stores the box with TMA while the warpgroup
    // fills the other buffer and then goes back to the next tile's wgmmas.  A 16-bit addend is loaded into the buffers
    // by TMA behind mbarriers (the first two chunks during the tile's mainloop), an fp32 accumulation (C == D) is
    // issued as a TMA reduce-add, so the epilogue loads nothing from global memory but the bias.
    const uint32_t stage_buf = bar_base + S::kBarrierBytes + wg * 16384;   // + b * 8192, b = chunk & 1
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const bool stage_addend = kStaged && args.C != nullptr && !args.out_fp32;   // fp32 C is always C == D (host)
    auto cload_bar = [&](int b) { return bar_base + 8u * (2 * kStages + 2 * wg + b); };
    auto load_addend = [&](int chunk, int tm, int tn) {   // wg_leader only, buffer (chunk & 1) free
      const int b = chunk & 1;
      mbar_arrive_expect_tx(cload_bar(b), 8192);
      tma_load_2d(stage_buf + b * 8192, &maps.c, cload_bar(b), tn * kBlockN + 64 * chunk, tm * kBlockM + wg * 64);
    };
    int it = 0;
    for (int t = cta; t < num_tiles; t += num_ctas) {
      int tm, tn, shard;
      coords(t, tm, tn, shard);
      int nkb = num_k_blocks, k_base;
      if constexpr (kGroup == 2) {
        nkb = expert_k_blocks(shard, k_base);
        if (nkb == 0) {   // expert without rows: its gradient is zero; when accumulating, D stays as it is
          if (args.C == nullptr) {
            const int col = tn * kBlockN + (int)(threadIdx.x - 128);
            for (int r = 0; r < kBlockM && col < args.N; ++r) {
              const long long row = (long long)tm * kBlockM + r;
              if (row >= args.M) break;
              const long long off = ((long long)shard * args.M + row) * args.ldd + col;
              if (args.out_fp32) reinterpret_cast<float*>(args.D)[off] = 0.f;
              else reinterpret_cast<uint16_t*>(args.D)[off] = 0;
            }
          }
          continue;
        }
      }
      float acc[kBlockN / 2];
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % kStages;
        mbar_wait(full_bar(s), (it / kStages) & 1);
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          const uint64_t da = (kAMajor == Major::K) ? desc_kmajor_sw128(smem_a(s) + wg * 8192, k)
                                                     : desc_mnmajor_sw128(smem_a(s) + wg * 8192, k, 8192);
          const uint64_t db = (kBMajor == Major::K) ? desc_kmajor_sw128(smem_b(s), k)
                                                     : desc_mnmajor_sw128(smem_b(s), k, 8192);
          wgmma_ss<kBlockN, kBf16, kTA, kTB>(acc, da, db, (kb | k) != 0);
        }
        wgmma_commit();
        if (kb > 0) {   // the MMAs of the previous K block have retired: hand its smem slot back to the producer
          wgmma_wait<1>();
          if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar((it - 1) % kStages));
        }
        if constexpr (kStaged) {
          // addend chunks 0 and 1 of this tile, once the previous tile's stores have left the staging buffers
          if (stage_addend && wg_leader && kb == min(nkb - 1, 1)) {
            tma_store_wait_read<0>();
            load_addend(0, tm, tn);
            load_addend(1, tm, tn);
          }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar((it - 1) % kStages));

      const long long row0 = (long long)tm * kBlockM + frag_row;   // this thread's rows: row0 and row0 + 8
      if constexpr (kStaged) {
        // Fragment element (row r + 8 half, column 8 j + 2 quad + e) of the warpgroup's 64 rows.  A 16-bit chunk is
        // 64 columns (j in [8c, 8c + 8)): each pair is one 32-bit word in 16-byte unit j % 8 of its 128-byte row.  An
        // fp32 chunk is 32 columns (j in [4c, 4c + 4)): each pair is 8 bytes in unit 2 (j % 4) + quad / 2.  The
        // 128-byte swizzle XORs the unit with the row's index mod 8.
        const uint32_t r = (uint32_t)(wq * 16) + (lane >> 2);
        auto addr16 = [&](int b, int jj, int half) {
          const uint32_t row = r + 8u * half;
          return stage_buf + b * 8192 + row * 128u + (((uint32_t)jj ^ (row & 7u)) << 4) + quad * 4u;
        };
        auto addr32 = [&](int b, int jj, int half) {
          const uint32_t row = r + 8u * half;
          return stage_buf + b * 8192 + row * 128u + (((uint32_t)(2 * jj) + (quad >> 1)) ^ (row & 7u)) * 16u +
                 (quad & 1u) * 8u;
        };
        const int mrow = tm * kBlockM + wg * 64;
        auto wg_sync = [&]() { named_bar_sync(1 + wg, 128); };
        auto acquire = [&]() {   // this chunk's buffer is free again: the store two chunks back has read it
          if (wg_leader) tma_store_wait_read<1>();
          wg_sync();
        };
        auto release = [&]() {   // generic-proxy writes -> visible to the TMA store, all 128 threads done
          fence_proxy_async_smem();
          wg_sync();
        };
        auto store16 = [&](const CUtensorMap* map, int b, int col) {
          release();
          if (wg_leader) {
            tma_store_2d(map, stage_buf + b * 8192, col, mrow);
            tma_store_commit();
          }
        };
        if (args.swiglu) {
          // h chunks 0, 1, then (with gu_out) g chunks 0, 1 and u chunks 0, 1; same arithmetic as the register path
          const int hcol = tn * (kBlockN / 2);
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            acquire();
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * c + jj;
#pragma unroll
              for (int half = 0; half < 2; ++half) {
                float hv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float gt = acc[4 * j + 2 * half + e], up = acc[4 * (j + 16) + 2 * half + e];
                  hv[e] = gt * fast_sigmoid(gt) * up;
                }
                st_shared_b32(addr16(c, jj, half), pk(hv[0], hv[1]));
              }
            }
            store16(&maps.d, c, hcol + 64 * c);
          }
          if (args.gu_out != nullptr) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {   // c < 2: gate columns, c >= 2: up columns (accumulator columns + 128)
              const int b = c & 1, jo = (c >> 1) * 16 + 8 * b;
              acquire();
#pragma unroll
              for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int half = 0; half < 2; ++half)
                  st_shared_b32(addr16(b, jj, half), pk(acc[4 * (jo + jj) + 2 * half], acc[4 * (jo + jj) + 2 * half + 1]));
              store16(&maps.gu, b, (c >> 1) * args.swiglu_F + hcol + 64 * b);
            }
          }
          continue;
        }
        const int n0 = tn * kBlockN;
        const uint16_t* bias = reinterpret_cast<const uint16_t*>(args.bias);
        if (args.out_fp32) {
          // fp32: 8 chunks of 32 columns; accumulation (C == D) adds the staged tile with a TMA reduce-add, which is
          // old + (acc + b) where the register path computes (acc + b) + old: the same IEEE sum
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const int b = c & 1;
            acquire();
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * c + jj;
              const int col = n0 + 8 * j + 2 * (int)quad;
              const float b0 = (bias && col < args.N) ? ld1(bias + col) : 0.f;
              const float b1 = (bias && col + 1 < args.N) ? ld1(bias + col + 1) : 0.f;
#pragma unroll
              for (int half = 0; half < 2; ++half)
                st_shared_v2_f32(addr32(b, jj, half), acc[4 * j + 2 * half] + b0, acc[4 * j + 2 * half + 1] + b1);
            }
            release();
            if (wg_leader) {
              if (args.C != nullptr) tma_reduce_add_2d(&maps.d, stage_buf + b * 8192, n0 + 32 * c, mrow);
              else tma_store_2d(&maps.d, stage_buf + b * 8192, n0 + 32 * c, mrow);
              tma_store_commit();
            }
          }
          continue;
        }
        // 16-bit: 4 chunks of 64 columns; bias and addend in fp32 in the accumulator layout, then one rounding
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int b = c & 1;
          if (stage_addend) mbar_wait(cload_bar(b), (c >> 1) & 1);
          else acquire();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * c + jj;
            const int col = n0 + 8 * j + 2 * (int)quad;
            float b0 = 0.f, b1 = 0.f;
            if (bias) {
              if (col < args.N) b0 = ld1(bias + col);
              if (col + 1 < args.N) b1 = ld1(bias + col + 1);
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
              if (bias) { v0 += b0; v1 += b1; }
              if (stage_addend) {
                const float2 old = unpack_h2<kBf16>(ld_shared_b32(addr16(b, jj, half)));
                v0 += old.x; v1 += old.y;
              }
              st_shared_b32(addr16(b, jj, half), pk(v0, v1));
            }
          }
          store16(&maps.d, b, n0 + 64 * c);
          if (stage_addend && wg_leader && c + 2 < 4) {   // addend chunk c + 2 into this buffer once it is read out
            tma_store_wait_read<0>();
            load_addend(c + 2, tm, tn);
          }
        }
        continue;
      }
      if constexpr (kFuse == 2) {
        // bf16 partial tile -> staging slot [my rank] of the rank that owns this row block (peer stores over NVLink,
        // 16 bytes per lane after the quad transpose); slots are row-major [rows_per_rank][N padded to the tile].
        if (shard != cur_shard) {
          flush_arrivals();
          cur_shard = shard;
        }
        const long long npad = (long long)args.num_n_tiles * kBlockN;
        uint16_t* slot = reinterpret_cast<uint16_t*>(args.fuse.peer[shard]) + (long long)args.fuse.rank * args.fuse.slot_stride;
        const long long lrow0 = row0 - (long long)shard * args.fuse.rows_per_rank;
#pragma unroll
        for (int g = 0; g < kBlockN / 32; ++g) {
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            uint32_t x[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) x[jj] = pack_bf16x2(acc[4 * (4 * g + jj) + 2 * half], acc[4 * (4 * g + jj) + 2 * half + 1]);
            quad_transpose(x, lane);
            const int col = tn * kBlockN + 32 * g + 8 * (int)quad;
            if (col + 8 <= args.N)
              *reinterpret_cast<uint4*>(slot + (lrow0 + 8 * half) * npad + col) = make_uint4(x[0], x[1], x[2], x[3]);
          }
        }
        ++pending;
        continue;
      }
      if constexpr (kFuse == 0) {
        if (args.swiglu) {
          const bool vec_h = true;   // F % 128 == 0 and the row pitches are multiples of 8 elements (checked on the host)
#pragma unroll
          for (int g = 0; g < 4; ++g) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              uint32_t xh[4], xg[4], xu[4];
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * g + jj;
                float hv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float gt = acc[4 * j + 2 * half + e], up = acc[4 * (j + 16) + 2 * half + e];
                  hv[e] = gt * fast_sigmoid(gt) * up;
                }
                xh[jj] = pk(hv[0], hv[1]);
                xg[jj] = pk(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
                xu[jj] = pk(acc[4 * (j + 16) + 2 * half], acc[4 * (j + 16) + 2 * half + 1]);
              }
              quad_transpose(xh, lane);
              const long long grow = row0 + 8 * half;
              const int col = tn * (kBlockN / 2) + 32 * g + 8 * (int)quad;   // output column (of F)
              const bool ok = grow < args.M && col < args.swiglu_F;
              if (ok) store_row8(reinterpret_cast<uint16_t*>(args.D) + grow * args.ldd + col, xh, args.swiglu_F - col, vec_h);
              if (args.gu_out != nullptr) {
                quad_transpose(xg, lane);
                quad_transpose(xu, lane);
                if (ok) {
                  uint16_t* gp = reinterpret_cast<uint16_t*>(args.gu_out) + grow * args.ldgu + col;
                  store_row8(gp, xg, args.swiglu_F - col, vec_h);
                  store_row8(gp + args.swiglu_F, xu, args.swiglu_F - col, vec_h);
                }
              }
            }
          }
          continue;
        }
      }
      const int n0 = tn * kBlockN;
      const uint16_t* bias = reinterpret_cast<const uint16_t*>(args.bias);
      // grouped wgrad: expert `shard` owns rows [shard * M, shard * M + M) of D (and of C); 0 for every other mode
      const long long erow = (kGroup == 2) ? (long long)shard * args.M : 0;
      if (args.out_fp32) {
        // fp32 output: the four lanes of a quad already cover 32 contiguous bytes of a row
        const bool vec = (args.ldd % 2 == 0) && (args.C == nullptr || args.ldc % 2 == 0) &&
                         (reinterpret_cast<uintptr_t>(args.D) % 8 == 0) && (reinterpret_cast<uintptr_t>(args.C) % 8 == 0);
#pragma unroll
        for (int j = 0; j < kBlockN / 8; ++j) {
          const int col = n0 + 8 * j + 2 * (int)quad;
          if (col >= args.N) continue;
          const bool two = col + 1 < args.N;
          const float b0 = bias ? ld1(bias + col) : 0.f, b1 = (bias && two) ? ld1(bias + col + 1) : 0.f;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const long long grow = row0 + 8 * half;
            if (grow >= args.M) continue;
            float v0 = acc[4 * j + 2 * half] + b0, v1 = acc[4 * j + 2 * half + 1] + b1;
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
        // 16-bit output: bias / addend are applied in fp32 in the accumulator layout, then each quad transposes its
        // packed pairs so that every lane stores 16 contiguous bytes
        const bool vec_d = (args.ldd % 8 == 0) && (reinterpret_cast<uintptr_t>(args.D) % 16 == 0);
        const bool pair_c = args.C != nullptr && (args.ldc % 2 == 0) && (reinterpret_cast<uintptr_t>(args.C) % 4 == 0);
#pragma unroll
        for (int g = 0; g < kBlockN / 32; ++g) {
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
              if (row_ok && col < args.N) {
                const bool two = col + 1 < args.N;
                if (bias) {
                  v0 += ld1(bias + col);
                  if (two) v1 += ld1(bias + col + 1);
                }
                if (args.C) {
                  const uint16_t* cp = reinterpret_cast<const uint16_t*>(args.C) + (erow + grow) * args.ldc + col;
                  if (two && pair_c) {
                    const float2 old = unpack_h2<kBf16>(*reinterpret_cast<const uint32_t*>(cp));
                    v0 += old.x; v1 += old.y;
                  } else {
                    v0 += ld1(cp);
                    if (two) v1 += ld1(cp + 1);
                  }
                }
              }
              x[jj] = pk(v0, v1);
            }
            quad_transpose(x, lane);
            const int col = n0 + 32 * g + 8 * (int)quad;
            if (row_ok && col < args.N)
              store_row8(reinterpret_cast<uint16_t*>(args.D) + (erow + grow) * args.ldd + col, x, args.N - col, vec_d);
          }
        }
      }
    }
    flush_arrivals();
    if constexpr (kStaged) {
      if (wg_leader) tma_store_wait<0>();   // the staging buffers must outlive the stores that read them
    }
  }
  if constexpr (kFuse == 0) {
    if (args.carry.debug != nullptr && blockIdx.x == 0 && threadIdx.x == 0) args.carry.debug[7] = carry_now_ns();
  }
}

// ------------------------------------------------------------------------------------------------------
// Host launcher
// ------------------------------------------------------------------------------------------------------
template <bool kBf16, Major kAMajor, Major kBMajor, int kFuse, int kGroup = 0, bool kCarry = true, bool kStaged = false>
static cudaError_t launch_one(const CUtensorMap& ta, const CUtensorMap& tb_, const GemmArgs& args, int num_sms,
                              cudaStream_t stream, const EpiMaps& maps = EpiMaps{}) {
  using S = GemmSmem;
  auto kern = gemm_bf16_kernel<kBf16, kAMajor, kBMajor, kFuse, kGroup, kCarry, kStaged>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kStaged ? S::kTotalStaged : S::kTotalCarry);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  const bool carrying = kFuse == 0 && args.carry.slice[0].kind != 0;
  // grouped forward: the upper bound of row tiles (the real count is only known on the device)
  const int num_tiles = args.num_m_tiles * args.num_n_tiles * (kGroup == 2 ? args.group.num_experts : 1);
  const int comm_ctas = (kFuse == 1) ? args.fuse.comm_clusters * kCommCtasPerCluster : 0;
  int ctas = num_sms - comm_ctas;   // copy CTAs share their SMs with nobody
  if (ctas > num_tiles) ctas = num_tiles;
  if (ctas < 1) ctas = 1;
  ctas += comm_ctas;
  if (kFuse == 0 && args.dynamic) ctas = num_tiles;   // one CTA per tile: the block scheduler hands them to free SMs
  // the copy warp's ring only when there is something to carry, the staging buffers only for the staged epilogue
  const int smem = kStaged ? S::kTotalStaged : (carrying ? S::kTotalCarry : S::kTotal);
  kern<<<ctas, kNumThreads, smem, stream>>>(ta, tb_, args, maps);
  return cudaGetLastError();
}

// 1 = dynamic tile scheduling (one CTA per tile), 0 = static striping over a persistent grid.  mode < 0 only queries.
int gemm_sched_mode(int mode) {
  // default static; the sharding engine switches to dynamic when collectives run next to the GEMMs.
  // TORCHACC_B200_GEMM_SCHED=static|dynamic pins it.
  static int current = [] {
    const char* e = getenv("TORCHACC_B200_GEMM_SCHED");
    return (e && e[0] == 'd') ? 1 : 0;
  }();
  if (mode >= 0) current = mode ? 1 : 0;
  return current;
}

static bool fill_common(GemmArgs& args, void* D, const void* bias, int M, int N, int K, long long ldd, bool out_fp32,
                        const void* C, long long ldc) {
  args.D = D;
  args.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  args.M = M; args.N = N; args.K = K;
  args.ldd = ldd;
  args.C = C; args.ldc = ldc;
  args.out_fp32 = out_fp32 ? 1 : 0;
  args.num_m_tiles = (M + kBlockM - 1) / kBlockM;
  args.num_n_tiles = (N + kBlockN - 1) / kBlockN;
  args.dynamic = gemm_sched_mode(-1);
  args.swiglu = 0; args.swiglu_F = 0; args.gu_out = nullptr; args.ldgu = 0;
  memset(&args.fuse, 0, sizeof(args.fuse));
  memset(&args.carry, 0, sizeof(args.carry));
  memset(&args.group, 0, sizeof(args.group));
  return true;
}

// K-major: matrix [MN][K], box 64 x box_rows; MN-major: matrix [K][MN], box 64 (MN) x 64 (K).  Inner box = 128 B.
static CUtensorMap operand_map(const void* p, int mn, int K, long long ld, bool mn_major, int box_rows) {
  return mn_major ? make_map_2d_bf16(p, K, mn, ld, 64, kBlockK) : make_map_2d_bf16(p, mn, K, ld, kBlockK, box_rows);
}

cudaError_t gemm_bf16(const void* A, const void* B, void* D, const void* bias, int M, int N, int K, long long lda,
                      long long ldb, long long ldd, bool a_mn_major, bool b_mn_major, bool out_fp32, bool accumulate,
                      int cluster, int num_sms, cudaStream_t stream, bool is_fp16) {
  return gemm_bf16_ex(A, B, D, bias, accumulate ? D : nullptr, M, N, K, lda, ldb, ldd, ldd, a_mn_major, b_mn_major,
                      out_fp32, cluster, num_sms, stream, is_fp16);
}

// K == 0: the product is empty, so D = bias (+ C) with the epilogue's arithmetic (an fp32 sum starting from a zero
// accumulator, one rounding): zeros without bias or addend, D unchanged when accumulating (C == D).  This is the weight
// gradient of a linear layer on an empty token batch.
template <bool kBf16>
__global__ void __launch_bounds__(256)
gemm_empty_k_kernel(void* D, const uint16_t* bias, const void* C, int M, int N, long long ldd, long long ldc, int out_fp32) {
  auto ld1 = [](const uint16_t* p) {
    return kBf16 ? __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p))
                 : __half2float(*reinterpret_cast<const __half*>(p));
  };
  const long long total = (long long)M * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / N;
    const int c = (int)(i - r * N);
    float v = 0.f;
    if (bias) v += ld1(bias + c);
    if (out_fp32) {
      if (C) v += reinterpret_cast<const float*>(C)[r * ldc + c];
      reinterpret_cast<float*>(D)[r * ldd + c] = v;
    } else {
      if (C) v += ld1(reinterpret_cast<const uint16_t*>(C) + r * ldc + c);
      reinterpret_cast<uint16_t*>(D)[r * ldd + c] = (uint16_t)(pack_h2<kBf16>(v, 0.f) & 0xffffu);
    }
  }
}

cudaError_t gemm_bf16_ex(const void* A, const void* B, void* D, const void* bias, const void* C, int M, int N, int K,
                         long long lda, long long ldb, long long ldd, long long ldc, bool a_mn_major, bool b_mn_major,
                         bool out_fp32, int cluster, int num_sms, cudaStream_t stream, bool is_fp16) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K < 0) return cudaErrorInvalidValue;
  if (cluster != 1 && cluster != 2) return cudaErrorInvalidValue;
  if (K == 0) {
    long long blocks = ((long long)M * N + 255) / 256;
    if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
    if (blocks < 1) blocks = 1;
    const uint16_t* b16 = reinterpret_cast<const uint16_t*>(bias);
    if (is_fp16) gemm_empty_k_kernel<false><<<(unsigned)blocks, 256, 0, stream>>>(D, b16, C, M, N, ldd, ldc, out_fp32);
    else gemm_empty_k_kernel<true><<<(unsigned)blocks, 256, 0, stream>>>(D, b16, C, M, N, ldd, ldc, out_fp32);
    return cudaGetLastError();
  }
  CUtensorMap ta, tbm;
  try {
    ta = operand_map(A, M, K, lda, a_mn_major, kBlockM);
    tbm = operand_map(B, N, K, ldb, b_mn_major, kBlockN / 2);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, D, bias, M, N, K, ldd, out_fp32, C, ldc);
  // pending FSDP collectives ride along: bytes proportional to this GEMM's FLOPs (static scheduling only -- under
  // dynamic scheduling the collectives run as their own kernels)
  if (!args.dynamic) carry_take(2.0 * (double)M * (double)N * (double)K, &args.carry);
  const bool carrying = args.carry.slice[0].kind != 0;
  // The staged (TMA) epilogue needs D and C 16-byte aligned with row pitches of whole 16 bytes; an fp32 addend is
  // only staged as an accumulation (C == D, TMA reduce-add).  Everything else keeps the register epilogue.
  // Rows must also end on a 16-byte boundary: at N * esz % 16 != 0 the TMA stores of a row's last box were measured
  // writing on to that boundary on an H100, up to 7 elements past N into the caller's pitch gap.
  const long long esz = out_fp32 ? 4 : 2;
  auto aligned = [&](const void* p, long long ld) { return reinterpret_cast<uintptr_t>(p) % 16 == 0 && (ld * esz) % 16 == 0; };
  const bool staged = !carrying && (N * esz) % 16 == 0 && aligned(D, ldd) &&
                      (C == nullptr || (out_fp32 ? (C == D && ldc == ldd) : aligned(C, ldc)));
  EpiMaps maps;
  memset(&maps, 0, sizeof(maps));
  if (staged) {
    try {
      maps.d = out_fp32 ? make_map_2d_f32(D, M, N, ldd, 32, 64) : make_map_2d_bf16(D, M, N, ldd, 64, 64);
      if (C != nullptr && !out_fp32) maps.c = make_map_2d_bf16(C, M, N, ldc, 64, 64);
    } catch (const std::exception& e) {
      fprintf(stderr, "%s\n", e.what());
      return cudaErrorInvalidValue;
    }
  }

#define TB_DISPATCH(BF, AM, BM)                                                                       \
  {                                                                                                   \
    if (carrying) return launch_one<BF, AM, BM, 0>(ta, tbm, args, num_sms, stream);                   \
    if (staged) return launch_one<BF, AM, BM, 0, 0, false, true>(ta, tbm, args, num_sms, stream, maps); \
    return launch_one<BF, AM, BM, 0, 0, false>(ta, tbm, args, num_sms, stream);                       \
  }
#define TB_MAJORS(BF)                                                  \
  if (!a_mn_major && !b_mn_major) TB_DISPATCH(BF, Major::K, Major::K); \
  if (!a_mn_major && b_mn_major) TB_DISPATCH(BF, Major::K, Major::MN); \
  if (a_mn_major && !b_mn_major) TB_DISPATCH(BF, Major::MN, Major::K); \
  TB_DISPATCH(BF, Major::MN, Major::MN)
  if (is_fp16) {
    TB_MAJORS(false);
  }
  TB_MAJORS(true);
#undef TB_MAJORS
#undef TB_DISPATCH
}

// h[M][F] = silu(x Wg^T) * (x Wu^T) with W_gu = [Wg; Wu] ([2F][K], K-major); optionally also gu[M][2F] = x W_gu^T.
cudaError_t gemm_swiglu_bf16(const void* A, const void* Wgu, void* H, void* GU, int M, int F, int K, long long lda,
                             long long ldb, long long ldh, long long ldgu, int num_sms, cudaStream_t stream,
                             bool is_fp16) {
  if (M <= 0 || F <= 0) return cudaSuccess;
  if (K <= 0 || F % 128 != 0 || ldh % 8 != 0 || (GU != nullptr && ldgu % 8 != 0)) return cudaErrorInvalidValue;
  if (reinterpret_cast<uintptr_t>(H) % 16 != 0 || reinterpret_cast<uintptr_t>(GU) % 16 != 0) return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_bf16(A, M, K, lda, kBlockK, kBlockM);
    tbm = make_map_2d_bf16(Wgu, 2 * (uint64_t)F, K, ldb, kBlockK, kBlockN / 2);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, H, nullptr, M, F, K, ldh, false, nullptr, 0);
  args.num_n_tiles = F / 128;           // each 256-wide accumulator tile yields 128 output columns
  args.swiglu = 1; args.swiglu_F = F; args.gu_out = GU; args.ldgu = ldgu;
  args.dynamic = 0;
  carry_take(4.0 * (double)M * (double)F * (double)K, &args.carry);
  if (args.carry.slice[0].kind != 0) {
    if (is_fp16) return launch_one<false, Major::K, Major::K, 0>(ta, tbm, args, num_sms, stream);
    return launch_one<true, Major::K, Major::K, 0>(ta, tbm, args, num_sms, stream);
  }
  // H and g|u are 16-byte aligned with whole-16-byte pitches (checked above): always the staged epilogue
  EpiMaps maps;
  memset(&maps, 0, sizeof(maps));
  try {
    maps.d = make_map_2d_bf16(H, M, F, ldh, 64, 64);
    if (GU != nullptr) maps.gu = make_map_2d_bf16(GU, M, 2 * (uint64_t)F, ldgu, 64, 64);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  if (is_fp16) return launch_one<false, Major::K, Major::K, 0, 0, false, true>(ta, tbm, args, num_sms, stream, maps);
  return launch_one<true, Major::K, Major::K, 0, 0, false, true>(ta, tbm, args, num_sms, stream, maps);
}

// ------------------------------------------------------------------------------------------------------
// Grouped (mixture-of-experts) entry points (see the GroupArgs comment).  No carried collectives ride along.
// ------------------------------------------------------------------------------------------------------
cudaError_t gemm_grouped_bf16(const void* A, const void* B, void* D, int M, int N, int K, int E, long long lda,
                              long long ldb, long long ldd, bool b_mn_major, const int* tile_expert,
                              const int* num_m_tiles, int num_sms, cudaStream_t stream, bool is_fp16) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K <= 0 || E <= 0 || M % kBlockM != 0 || tile_expert == nullptr || num_m_tiles == nullptr)
    return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = operand_map(A, M, K, lda, false, kBlockM);
    tbm = b_mn_major ? operand_map(B, N, E * K, ldb, true, kBlockN / 2)
                     : operand_map(B, E * N, K, ldb, false, kBlockN / 2);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, D, nullptr, M, N, K, ldd, false, nullptr, 0);
  args.dynamic = 0;
  args.group.tile_expert = tile_expert;
  args.group.num_m_tiles = num_m_tiles;
  args.group.b_rows = b_mn_major ? K : N;
  if (is_fp16) {
    if (b_mn_major) return launch_one<false, Major::K, Major::MN, 0, 1>(ta, tbm, args, num_sms, stream);
    return launch_one<false, Major::K, Major::K, 0, 1>(ta, tbm, args, num_sms, stream);
  }
  if (b_mn_major) return launch_one<true, Major::K, Major::MN, 0, 1>(ta, tbm, args, num_sms, stream);
  return launch_one<true, Major::K, Major::K, 0, 1>(ta, tbm, args, num_sms, stream);
}

cudaError_t gemm_grouped_swiglu_bf16(const void* A, const void* Wgu, void* H, void* GU, int M, int F, int K, int E,
                                     long long lda, long long ldb, long long ldh, long long ldgu,
                                     const int* tile_expert, const int* num_m_tiles, int num_sms, cudaStream_t stream,
                                     bool is_fp16) {
  if (M <= 0 || F <= 0) return cudaSuccess;
  if (K <= 0 || E <= 0 || M % kBlockM != 0 || F % 128 != 0 || ldh % 8 != 0 || (GU != nullptr && ldgu % 8 != 0))
    return cudaErrorInvalidValue;
  if (reinterpret_cast<uintptr_t>(H) % 16 != 0 || reinterpret_cast<uintptr_t>(GU) % 16 != 0) return cudaErrorInvalidValue;
  if (tile_expert == nullptr || num_m_tiles == nullptr) return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_bf16(A, M, K, lda, kBlockK, kBlockM);
    tbm = make_map_2d_bf16(Wgu, 2 * (uint64_t)F * E, K, ldb, kBlockK, kBlockN / 2);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, H, nullptr, M, F, K, ldh, false, nullptr, 0);
  args.num_n_tiles = F / 128;
  args.swiglu = 1; args.swiglu_F = F; args.gu_out = GU; args.ldgu = ldgu;
  args.dynamic = 0;
  args.group.tile_expert = tile_expert;
  args.group.num_m_tiles = num_m_tiles;
  args.group.b_rows = 2 * F;
  if (is_fp16) return launch_one<false, Major::K, Major::K, 0, 1>(ta, tbm, args, num_sms, stream);
  return launch_one<true, Major::K, Major::K, 0, 1>(ta, tbm, args, num_sms, stream);
}

cudaError_t gemm_grouped_wgrad_bf16(const void* dY, const void* X, void* D, int M, int N, int E, int rows,
                                    long long lda, long long ldb, long long ldd, const int* offsets, bool out_fp32,
                                    bool accumulate, int num_sms, cudaStream_t stream, bool is_fp16) {
  if (M <= 0 || N <= 0 || E <= 0) return cudaSuccess;
  if (rows <= 0 || rows % kBlockM != 0 || offsets == nullptr) return cudaErrorInvalidValue;
  CUtensorMap ta, tbm;
  try {
    ta = operand_map(dY, M, rows, lda, true, kBlockM);
    tbm = operand_map(X, N, rows, ldb, true, kBlockN / 2);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, D, nullptr, M, N, rows, ldd, out_fp32, accumulate ? D : nullptr, ldd);
  args.dynamic = 0;
  args.group.offsets = offsets;
  args.group.num_experts = E;
  if (is_fp16) return launch_one<false, Major::MN, Major::MN, 0, 2>(ta, tbm, args, num_sms, stream);
  return launch_one<true, Major::MN, Major::MN, 0, 2>(ta, tbm, args, num_sms, stream);
}

// ------------------------------------------------------------------------------------------------------
// Fused tensor-parallel entry points
// ------------------------------------------------------------------------------------------------------
static cudaError_t check_fused(int world, int rows_per_rank, int N, int channel) {
  if (world < 2 || world > kMaxPeers || channel < 0 || channel >= 64) return cudaErrorInvalidValue;
  if (rows_per_rank % (kBlockM * 2) != 0) return cudaErrorInvalidValue;   // M tiles must not straddle ranks
  if (N % 8 != 0) return cudaErrorInvalidValue;
  return cudaSuccess;
}

cudaError_t ag_gemm_bf16(const uint64_t* peer_a_full, const uint64_t* pad_ptrs, void* a_full, const void* B, void* D,
                         const void* bias, int rows_per_rank, int N, int K, long long ldb, long long ldd,
                         bool b_mn_major, int rank, int world, uint32_t* flags, uint32_t flag_target,
                         uint32_t* block_counter, int channel, uint32_t epoch, int comm_clusters, int num_sms,
                         cudaStream_t stream) {
  cudaError_t e = check_fused(world, rows_per_rank, N, channel);
  if (e != cudaSuccess) return e;
  if (K % 8 != 0 || comm_clusters < 1 || comm_clusters * kCommCtasPerCluster >= num_sms) return cudaErrorInvalidValue;
  const int M = rows_per_rank * world;
  CUtensorMap ta, tbm;
  try {
    ta = make_map_2d_bf16(a_full, M, K, K, kBlockK, kBlockM);
    tbm = operand_map(B, N, K, ldb, b_mn_major, kBlockN / 2);
  } catch (const std::exception& ex) {
    fprintf(stderr, "%s\n", ex.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, D, bias, M, N, K, ldd, false, nullptr, 0);
  FuseArgs& f = args.fuse;
  for (int i = 0; i < world; ++i) {
    f.peer[i] = reinterpret_cast<void*>(peer_a_full[i]);
    f.pads[i] = reinterpret_cast<uint32_t*>(pad_ptrs[i]);
  }
  f.a_full = a_full; f.flags = flags; f.block_counter = block_counter;
  f.rank = rank; f.world = world; f.rows_per_rank = rows_per_rank; f.channel = channel;
  f.epoch = epoch; f.flag_target = flag_target; f.comm_clusters = comm_clusters;
  if (b_mn_major) return launch_one<true, Major::K, Major::MN, 1>(ta, tbm, args, num_sms, stream);
  return launch_one<true, Major::K, Major::K, 1>(ta, tbm, args, num_sms, stream);
}

cudaError_t gemm_rs_bf16(const void* A, const void* B, const uint64_t* peer_stage, const uint64_t* peer_counters,
                         const uint64_t* pad_ptrs, int rows_per_rank, int N, int K, long long lda, long long ldb,
                         bool a_mn_major, bool b_mn_major, int rank, int world, int channel, uint32_t epoch,
                         int num_sms, cudaStream_t stream) {
  cudaError_t e = check_fused(world, rows_per_rank, N, channel);
  if (e != cudaSuccess) return e;
  if (N % 32 != 0) return cudaErrorInvalidValue;
  const int M = rows_per_rank * world;
  CUtensorMap ta, tbm;
  try {
    ta = operand_map(A, M, K, lda, a_mn_major, kBlockM);
    tbm = operand_map(B, N, K, ldb, b_mn_major, kBlockN / 2);
  } catch (const std::exception& ex) {
    fprintf(stderr, "%s\n", ex.what());
    return cudaErrorInvalidValue;
  }
  GemmArgs args;
  fill_common(args, nullptr, nullptr, M, N, K, /*ldd=*/N, false, nullptr, 0);
  FuseArgs& f = args.fuse;
  for (int i = 0; i < world; ++i) {
    f.peer[i] = reinterpret_cast<void*>(peer_stage[i]);
    f.peer_cnt[i] = reinterpret_cast<uint32_t*>(peer_counters[i]);
    f.pads[i] = reinterpret_cast<uint32_t*>(pad_ptrs[i]);
  }
  f.rank = rank; f.world = world; f.rows_per_rank = rows_per_rank; f.channel = channel; f.epoch = epoch;
  f.slot_stride = (long long)rows_per_rank * ((N + kBlockN - 1) / kBlockN * kBlockN);   // row-major, padded N
#define TB_RS(AM, BM) return launch_one<true, AM, BM, 2>(ta, tbm, args, num_sms, stream)
  if (!a_mn_major && !b_mn_major) TB_RS(Major::K, Major::K);
  if (!a_mn_major && b_mn_major) TB_RS(Major::K, Major::MN);
  if (a_mn_major && !b_mn_major) TB_RS(Major::MN, Major::K);
  TB_RS(Major::MN, Major::MN);
#undef TB_RS
}

// out[rows, N] = sum_src stage[src] (+ residual), once every source has delivered `expected` arrivals.
// Staging slots are row-major with the row pitch padded to the GEMM's 256-column tile; one thread sums 8 columns.
__global__ void __launch_bounds__(256)
rs_reduce_kernel(const __nv_bfloat16* __restrict__ stage, const uint32_t* __restrict__ counters, uint32_t expected,
                 const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ out, int rows, int N, int world,
                 long long slot_stride) {
  if (threadIdx.x < world)
    spin_until_count(counters + threadIdx.x, expected, -1, (int)threadIdx.x, "GEMM -> reduce-scatter arrivals");
  __syncthreads();
  const long long npad = (long long)((N + kBlockN - 1) / kBlockN) * kBlockN;
  const int vecs = N / 8;
  const long long total = (long long)rows * vecs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vecs;
    const int col = (int)(i % vecs) * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    auto add = [&](const uint4& u) {
      float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
      acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
      acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
    };
    for (int s = 0; s < world; ++s) add(ld_volatile_v4(stage + s * slot_stride + row * npad + col));
    if (residual) add(*reinterpret_cast<const uint4*>(residual + row * N + col));
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + row * N + col) = o;
  }
}

cudaError_t rs_reduce_bf16(const void* stage, const uint32_t* counters, uint32_t expected, const void* residual,
                           void* out, int rows, int N, int world, long long slot_stride, int num_sms,
                           cudaStream_t stream) {
  if (N % 32 != 0 || rows % 256 != 0) return cudaErrorInvalidValue;
  long long blocks = ((long long)rows * (N / 8) + 255) / 256;
  if (blocks > (long long)num_sms * 4) blocks = (long long)num_sms * 4;
  if (blocks < 1) blocks = 1;
  rs_reduce_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const __nv_bfloat16*)stage, counters, expected,
                                                          (const __nv_bfloat16*)residual, (__nv_bfloat16*)out, rows, N,
                                                          world, slot_stride);
  return cudaGetLastError();
}

}  // namespace tb
