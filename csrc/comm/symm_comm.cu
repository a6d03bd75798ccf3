// Symmetric-memory communication runtime for one NVSwitch domain (<= 8 GPUs per process group).
//
// Every rank allocates its communication buffers with cudaMalloc, exports them as CUDA IPC handles (exchanged through
// torch.distributed by the Python side) and maps every peer's buffer into its own address space.  Collectives are
// then plain CUDA kernels that read peer memory over NVLink with 16-byte loads ("pull"), synchronised by
// epoch-numbered flags in a small symmetric signal pad -- no NCCL on these paths:
//
//   all_gather      out[r*n:(r+1)*n] = peer_r.shard                        (FSDP parameter gather, TP activation gather)
//   reduce_scatter  out = scale * sum_r peer_r.buf[rank*n:(rank+1)*n]      (bf16 on the wire, fp32 accumulate/output)
//   all_reduce      in place, one-shot (every rank reduces everything) or two-shot (reduce-scatter + all-gather)
//   all_to_all      out[r*c:(r+1)*c] = peer_r.buf[rank*c:(rank+1)*c]       (Ulysses head/sequence exchange)
//
// Protocol per call (epoch e, channel ch):  entry barrier  (everybody's input is in place)  ->  pull  ->
// exit barrier (everybody finished reading my buffer, so it may be overwritten).  The barriers are device side:
// block 0 publishes `e` into slot [ch][my_rank] of every peer's pad (st.release.sys) and all blocks spin on their own
// pad (ld.acquire.sys) -- the spin is on LOCAL memory.
//
// Replaces: NCCL all-gather / reduce-scatter / all-reduce / all-to-all calls the reference makes through torch FSDP,
// DDP and torch.distributed (SURVEY 2.4b).
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../common/ptx.cuh"
#include "../common/spin.cuh"
#include "comm.h"

namespace tb {

constexpr int kMaxWorld = 8;
constexpr int kPadChannels = 64;
constexpr int kPadSlots = 16;  // per channel: [0,8) entry flags, [8,16) exit flags

struct Peers {
  void* ptr[kMaxWorld];
};
struct Pads {
  uint32_t* ptr[kMaxWorld];
};

TB_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
TB_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Streaming access for the collectives' bulk traffic.  Loads are strong (relaxed.sys: never served from a stale L1
// line -- the same addresses are rewritten by other SMs / GPUs every step) and do not allocate in L1; loads and stores
// carry an L2 evict-first policy.  Without it the ~2 GB a collective streams per layer flushes the operand tiles the
// concurrently running GEMMs keep L2-resident and slows every GEMM that overlaps a collective.
TB_DEVICE uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
TB_DEVICE uint4 ld_stream_v4(const void* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol)
               : "memory");
  return v;
}
TB_DEVICE void st_stream_v4(void* p, const uint4& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w), "l"(pol)
               : "memory");
}
TB_DEVICE void st_stream_v2(void* p, const uint2& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.u32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol) : "memory");
}

// Entry barrier: all ranks have launched this collective and their inputs are written.
TB_DEVICE void barrier_enter(const Pads& pads, int rank, int world, int ch, uint32_t epoch) {
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(pads.ptr[threadIdx.x] + ch * kPadSlots + rank, epoch);
  }
  if (threadIdx.x < world)
    spin_until_epoch(pads.ptr[rank] + ch * kPadSlots + threadIdx.x, epoch, rank, (int)threadIdx.x, ch, "collective entry");
  __syncthreads();
}

// Exit barrier: every block of THIS rank is done reading, then tell the peers; block 0 stays until all peers are done.
TB_DEVICE void barrier_exit(const Pads& pads, int rank, int world, int ch, uint32_t epoch, uint32_t* block_counter) {
  __syncthreads();
  __shared__ uint32_t s_last;
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t prev = atomicAdd(block_counter, 1u);
    s_last = (prev == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) *block_counter = 0;  // re-arm for the next call (stream ordered)
  if (threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(pads.ptr[threadIdx.x] + ch * kPadSlots + 8 + rank, epoch);
    spin_until_epoch(pads.ptr[rank] + ch * kPadSlots + 8 + threadIdx.x, epoch, rank, (int)threadIdx.x, ch,
                     "collective exit");
  }
  __syncthreads();
}

// ----------------------------------------------------------------------------------------------------------
// all-gather (bytes): out + r*bytes <- peer[r] (+ src_off)
// ----------------------------------------------------------------------------------------------------------
// Register budget: 32 registers x 512 threads, a quarter of an SM's register file, so four CTAs fit on an SM.  On sm_90a a
// wgmma GEMM CTA (384 threads, 168 registers each before setmaxnreg) owns the whole register file of its SM, so a
// collective CTA and a GEMM CTA never share an SM: collectives take SMs from a concurrently running GEMM, which then
// uses dynamic scheduling (gemm_sched_mode).  How well the two overlap on H100 has not been measured.
__global__ void __launch_bounds__(512, 4)
all_gather_kernel(const __grid_constant__ Peers src, const __grid_constant__ Pads pads, uint8_t* __restrict__ out,
                  size_t bytes, int rank, int world, int ch, uint32_t epoch, uint32_t* block_counter) {
  barrier_enter(pads, rank, world, ch, epoch);
  const uint64_t pol = l2_evict_first_policy();
  const uint32_t nvec = (uint32_t)(bytes >> 4);                 // < 2^31 vectors (32 GB) per shard
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int step = 0; step < world; ++step) {
    const int r = (rank + step) % world;  // start with the local shard, then walk the ring so peers are hit evenly
    const uint4* s = reinterpret_cast<const uint4*>(src.ptr[r]);
    uint4* d = reinterpret_cast<uint4*>(out + (size_t)r * bytes);
    if (r == rank && (const void*)s == (const void*)d) continue;  // shard already lives inside the output buffer
    uint32_t i = tid;
    for (; i + 3 * stride < nvec; i += 4 * stride) {
      const uint4 a = ld_stream_v4(s + i, pol), b = ld_stream_v4(s + i + stride, pol),
                  c = ld_stream_v4(s + i + 2 * stride, pol), e = ld_stream_v4(s + i + 3 * stride, pol);
      st_stream_v4(d + i, a, pol); st_stream_v4(d + i + stride, b, pol);
      st_stream_v4(d + i + 2 * stride, c, pol); st_stream_v4(d + i + 3 * stride, e, pol);
    }
    for (; i < nvec; i += stride) st_stream_v4(d + i, ld_stream_v4(s + i, pol), pol);
  }
  barrier_exit(pads, rank, world, ch, epoch, block_counter);
}

// ----------------------------------------------------------------------------------------------------------
// reduce-scatter: out[i] = scale * sum_r peer_r[rank*n + i], fp32 accumulation.  In: bf16 or fp32.  Out: fp32/bf16.
// ----------------------------------------------------------------------------------------------------------
template <typename InT, typename OutT>
__global__ void __launch_bounds__(512, 3)
reduce_scatter_kernel(const __grid_constant__ Peers src, const __grid_constant__ Pads pads, OutT* __restrict__ out, size_t n, float scale, int rank, int world, int ch,
                      uint32_t epoch, uint32_t* block_counter) {
  barrier_enter(pads, rank, world, ch, epoch);
  const uint64_t pol = l2_evict_first_policy();
  constexpr int kPer = 16 / sizeof(InT);  // elements per 16-byte load: 8 (bf16) or 4 (fp32)
  const size_t nvec = n / kPer;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float acc[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) acc[j] = 0.f;
    // four peers per batch: 4 loads in flight, 16 data registers (the kernel must stay small enough to share an SM
    // with a GEMM CTA and an all-gather CTA)
    for (int base = 0; base < world; base += 4) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (base + j < world) {
          const int r = (rank + base + j) % world;
          v[j] = ld_stream_v4(reinterpret_cast<const uint4*>(reinterpret_cast<const InT*>(src.ptr[r]) + (size_t)rank * n) + i, pol);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (base + j < world) {
          if constexpr (sizeof(InT) == 2) {
            float2 a = unpack_bf16x2(v[j].x), b = unpack_bf16x2(v[j].y), c = unpack_bf16x2(v[j].z),
                   d = unpack_bf16x2(v[j].w);
            acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
            acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
          } else {
            acc[0] += __uint_as_float(v[j].x); acc[1] += __uint_as_float(v[j].y);
            acc[2] += __uint_as_float(v[j].z); acc[3] += __uint_as_float(v[j].w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kPer; ++j) acc[j] *= scale;
    if constexpr (sizeof(OutT) == 4) {
      uint4* o = reinterpret_cast<uint4*>(out + i * kPer);
      st_stream_v4(o, make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]),
                                 __float_as_uint(acc[3])), pol);
      if constexpr (kPer == 8)
        st_stream_v4(o + 1, make_uint4(__float_as_uint(acc[4]), __float_as_uint(acc[5]), __float_as_uint(acc[6]),
                                       __float_as_uint(acc[7])), pol);
    } else {
      if constexpr (kPer == 8) {
        uint4 o;
        o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
        o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
        st_stream_v4(out + i * 8, o, pol);
      } else {
        uint2 o;
        o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
        st_stream_v2(out + i * 4, o, pol);
      }
    }
  }
  barrier_exit(pads, rank, world, ch, epoch, block_counter);
}

// ----------------------------------------------------------------------------------------------------------
// all-to-all (bytes): out + r*chunk <- peer[r] + rank*chunk
// ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512, 4)
all_to_all_kernel(const __grid_constant__ Peers src, const __grid_constant__ Pads pads, uint8_t* __restrict__ out, size_t chunk_bytes, int rank, int world, int ch,
                  uint32_t epoch, uint32_t* block_counter) {
  barrier_enter(pads, rank, world, ch, epoch);
  const uint64_t pol = l2_evict_first_policy();
  const size_t nvec = chunk_bytes >> 4;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (int step = 0; step < world; ++step) {
    const int r = (rank + step) % world;
    const uint4* s = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(src.ptr[r]) + (size_t)rank * chunk_bytes);
    uint4* d = reinterpret_cast<uint4*>(out + (size_t)r * chunk_bytes);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride)
      st_stream_v4(d + i, ld_stream_v4(s + i, pol), pol);
  }
  barrier_exit(pads, rank, world, ch, epoch, block_counter);
}

// ----------------------------------------------------------------------------------------------------------
// TMA variants (large messages).  Long-latency LSU requests to peer memory sit in the SM<->L2 fabric that a
// concurrently running GEMM's operand traffic uses; bulk-async copies do not.  So large collectives
// are driven by ONE thread per CTA issuing 32 KB `cp.async.bulk` transfers  peer HBM -> smem -> local HBM  (or smem ->
// 256 reducer threads for reduce-scatter).  A CTA keeps (stages-1) x 32 KB in flight, so <= 16 CTAs fill the link;
// the SMs they occupy (no co-residency with a GEMM CTA) receive no tiles from the GEMM's dynamic schedule.
// ----------------------------------------------------------------------------------------------------------
constexpr uint32_t kTmaChunk = 32768;
constexpr int kTmaStages = 6;
constexpr int kTmaSmem = kTmaStages * kTmaChunk + 1024 + 256;

struct CopyList {            // for each source rank r: copy `bytes` from src[r] to dst[r]
  const uint8_t* src[kMaxWorld];
  uint8_t* dst[kMaxWorld];
};

__global__ void __launch_bounds__(32)
multi_copy_tma_kernel(const __grid_constant__ CopyList cl, const __grid_constant__ Pads pads, size_t bytes, int rank,
                      int world, uint32_t kTmaChunk, uint32_t kTmaStages, int ch, uint32_t epoch,
                      uint32_t* block_counter) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
  const uint32_t bar = base + kTmaStages * kTmaChunk;
  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < kTmaStages; ++s) mbar_init(bar + 8u * s, 1);
    fence_mbar_init();
  }
  barrier_enter(pads, rank, world, ch, epoch);   // (ends with __syncthreads)
  if (threadIdx.x == 0) {
    asm volatile("fence.proxy.async;" ::: "memory");   // peers' generic-proxy writes (acquired above) -> TMA reads
    const uint32_t chunks = (uint32_t)((bytes + kTmaChunk - 1) / kTmaChunk);
    const uint32_t per = chunks > blockIdx.x ? (chunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    int nsrc = 0, order[kMaxWorld];
    for (int step = 0; step < world; ++step) {   // local shard first (if it needs copying), then the ring
      const int r = (rank + step) % world;
      if (cl.src[r] != cl.dst[r]) order[nsrc++] = r;
    }
    const uint32_t total = per * nsrc;
    auto locate = [&](uint32_t j, const uint8_t*& sp, uint8_t*& dp, uint32_t& len) {
      const int r = order[j / per];
      const size_t off = (size_t)(blockIdx.x + (j % per) * gridDim.x) * kTmaChunk;
      sp = cl.src[r] + off;
      dp = cl.dst[r] + off;
      const size_t left = bytes - off;
      len = left < kTmaChunk ? (uint32_t)left : kTmaChunk;
    };
    auto issue = [&](uint32_t j) {
      const uint8_t* sp; uint8_t* dp; uint32_t len;
      locate(j, sp, dp, len);
      const uint32_t st = j % kTmaStages;
      mbar_arrive_expect_tx(bar + 8u * st, len);
      bulk_load(base + st * kTmaChunk, sp, len, bar + 8u * st);
    };
    uint32_t issued = 0;
    for (; issued < kTmaStages - 1 && issued < total; ++issued) issue(issued);
    for (uint32_t i = 0; i < total; ++i) {
      const uint32_t st = i % kTmaStages;
      mbar_wait(bar + 8u * st, (i / kTmaStages) & 1);
      const uint8_t* sp; uint8_t* dp; uint32_t len;
      locate(i, sp, dp, len);
      bulk_store(dp, base + st * kTmaChunk, len);
      tma_store_commit();
      if (issued < total) {
        tma_store_wait_read<1>();     // all stores but the newest have left smem: stage (i-1) % stages is free
        issue(issued++);
      }
    }
    tma_store_wait<0>();              // writes complete before the exit barrier publishes "done"
  }
  barrier_exit(pads, rank, world, ch, epoch, block_counter);
}

// reduce-scatter: warps 0-7 reduce, warp 8 lane 0 produces.  Stage = `world` sub-chunks (one per source rank).
template <typename InT, typename OutT>
__global__ void __launch_bounds__(288, 1)
reduce_scatter_tma_kernel(const __grid_constant__ Peers src, const __grid_constant__ Pads pads, OutT* __restrict__ out,
                          size_t n, float scale, int rank, int world, uint32_t sub_bytes, int stages, int ch,
                          uint32_t epoch, uint32_t* block_counter) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t stage_bytes = sub_bytes * world;
  const uint32_t bar = base + stages * stage_bytes;      // full[s] at +8s, empty[s] at +8(stages+s)
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar + 8u * s, 1);
      mbar_init(bar + 8u * (stages + s), 8);              // one arrive per reducer warp
    }
    fence_mbar_init();
  }
  barrier_enter(pads, rank, world, ch, epoch);
  const size_t total_bytes = n * sizeof(InT);
  const uint32_t chunks = (uint32_t)((total_bytes + sub_bytes - 1) / sub_bytes);
  const uint32_t per = chunks > blockIdx.x ? (chunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  if (threadIdx.x == 256) {
    // ---- producer ----
    asm volatile("fence.proxy.async;" ::: "memory");
    for (uint32_t i = 0; i < per; ++i) {
      const uint32_t st = i % stages;
      if (i >= (uint32_t)stages) mbar_wait(bar + 8u * (stages + st), ((i / stages) - 1) & 1);
      const size_t off = (size_t)(blockIdx.x + i * gridDim.x) * sub_bytes;
      const size_t left = total_bytes - off;
      const uint32_t len = left < sub_bytes ? (uint32_t)left : sub_bytes;
      mbar_arrive_expect_tx(bar + 8u * st, len * world);
      for (int p = 0; p < world; ++p) {
        const int r = (rank + p) % world;
        const uint8_t* sp = reinterpret_cast<const uint8_t*>(src.ptr[r]) + (size_t)rank * total_bytes + off;
        bulk_load(base + st * stage_bytes + p * sub_bytes, sp, len, bar + 8u * st);
      }
    }
  } else if (threadIdx.x < 256) {
    // ---- reducers ----
    const uint64_t pol = l2_evict_first_policy();
    constexpr int kPer = 16 / sizeof(InT);
    for (uint32_t i = 0; i < per; ++i) {
      const uint32_t st = i % stages;
      mbar_wait(bar + 8u * st, (i / stages) & 1);
      const size_t off = (size_t)(blockIdx.x + i * gridDim.x) * sub_bytes;
      const size_t left = total_bytes - off;
      const uint32_t len = left < sub_bytes ? (uint32_t)left : sub_bytes;
      const uint32_t nvec = len >> 4;
      const uint32_t sbase = base + st * stage_bytes;
      OutT* o = out + off / sizeof(InT);
      for (uint32_t v = threadIdx.x; v < nvec; v += 256) {
        float acc[kPer];
#pragma unroll
        for (int j = 0; j < kPer; ++j) acc[j] = 0.f;
        for (int p = 0; p < world; ++p) {
          uint4 u;
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                       : "r"(sbase + p * sub_bytes + v * 16));
          if constexpr (sizeof(InT) == 2) {
            float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
            acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
            acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
          } else {
            acc[0] += __uint_as_float(u.x); acc[1] += __uint_as_float(u.y);
            acc[2] += __uint_as_float(u.z); acc[3] += __uint_as_float(u.w);
          }
        }
#pragma unroll
        for (int j = 0; j < kPer; ++j) acc[j] *= scale;
        if constexpr (sizeof(OutT) == 4) {
          uint4* op = reinterpret_cast<uint4*>(o + (size_t)v * kPer);
          st_stream_v4(op, make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]),
                                      __float_as_uint(acc[3])), pol);
          if constexpr (kPer == 8)
            st_stream_v4(op + 1, make_uint4(__float_as_uint(acc[4]), __float_as_uint(acc[5]), __float_as_uint(acc[6]),
                                            __float_as_uint(acc[7])), pol);
        } else {
          if constexpr (kPer == 8) {
            uint4 ov;
            ov.x = pack_bf16x2(acc[0], acc[1]); ov.y = pack_bf16x2(acc[2], acc[3]);
            ov.z = pack_bf16x2(acc[4], acc[5]); ov.w = pack_bf16x2(acc[6], acc[7]);
            st_stream_v4(o + (size_t)v * 8, ov, pol);
          } else {
            uint2 ov;
            ov.x = pack_bf16x2(acc[0], acc[1]); ov.y = pack_bf16x2(acc[2], acc[3]);
            st_stream_v2(o + (size_t)v * 4, ov, pol);
          }
        }
      }
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbar_arrive(bar + 8u * (stages + st));
    }
  }
  barrier_exit(pads, rank, world, ch, epoch, block_counter);
}

// ----------------------------------------------------------------------------------------------------------
// host API
// ----------------------------------------------------------------------------------------------------------
static int comm_cta_cap() {
  static int cap = [] {
    const char* e = getenv("TORCHACC_B200_COMM_CTAS");
    const int v = e ? atoi(e) : 0;
    return v > 0 ? v : 64;
  }();
  return cap;
}

static int grid_for(size_t bytes, int num_sms) {
  size_t blocks = (bytes / 16 + 511) / 512;
  // ~64 CTAs of 512 threads (4 x 16 B in flight per thread) saturate NVLink; the collectives run next to persistent
  // GEMMs, so fewer CTAs leave more issue slots / L2 bandwidth to the tensor-core kernels
  const int cap = num_sms < comm_cta_cap() ? num_sms : comm_cta_cap();
  if (blocks > (size_t)cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// The collectives run concurrently with wgmma GEMM CTAs that need the maximum shared-memory carve-out (~199 KB).
// An SM cannot host CTAs of two kernels with different L1/shared carve-outs, and changing the carve-out of an SM waits
// for it to drain: asking for the max-shared carve-out here lets an SM pass from a collective CTA to a GEMM CTA (and
// back) without that reconfiguration.
template <typename K>
static void prefer_max_smem_carveout(K kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
static void configure_kernels_once() {
  static bool done = [] {
    prefer_max_smem_carveout(all_gather_kernel);
    prefer_max_smem_carveout(all_to_all_kernel);
    prefer_max_smem_carveout(reduce_scatter_kernel<__nv_bfloat16, float>);
    prefer_max_smem_carveout(reduce_scatter_kernel<__nv_bfloat16, __nv_bfloat16>);
    prefer_max_smem_carveout(reduce_scatter_kernel<float, float>);
    prefer_max_smem_carveout(reduce_scatter_kernel<float, __nv_bfloat16>);
    return true;
  }();
  (void)done;
}

static int tma_min_bytes() {
  static int v = [] {
    const char* e = getenv("TORCHACC_B200_COMM_TMA_MIN");   // bytes; 0 disables the TMA collectives
    return e ? atoi(e) : (1 << 20);
  }();
  return v;
}
static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  const int n = e ? atoi(e) : dflt;
  return n > 0 ? n : dflt;
}
// reduce-scatter: CTAs with a 192 KB staging ring (they own their SM)
static int rs_ctas() {
  static int v = env_int("TORCHACC_B200_COMM_RS_CTAS", 16);
  return v;
}
// copy kernels (all-gather / all-to-all): many one-warp CTAs with a small ring (3 x 8 KB).  A CTA's bulk copies from
// peer memory do not pipeline deeper than ~32 KB, so bandwidth comes from the number of SMs driving TMA, not from ring
// depth.  The CTA count was chosen on another GPU and has not been re-derived for the 132 SMs of an H100.
static int tma_ctas() {
  static int v = env_int("TORCHACC_B200_COMM_TMA_CTAS", 120);
  return v;
}
static uint32_t copy_chunk() {
  static int v = env_int("TORCHACC_B200_COMM_TMA_CHUNK", 8192) & ~15;
  return (uint32_t)v;
}
static uint32_t copy_stages() {
  static int v = env_int("TORCHACC_B200_COMM_TMA_STAGES", 3);
  return (uint32_t)(v < 2 ? 2 : v);
}
static int copy_smem() { return (int)(copy_chunk() * copy_stages()) + 128 + 256; }
template <typename K>
static cudaError_t allow_smem(K kernel, int bytes) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

static void fill(Peers& p, Pads& q, const uint64_t* peer_ptrs, const uint64_t* pad_ptrs, int world, size_t off_bytes) {
  for (int i = 0; i < kMaxWorld; ++i) {
    p.ptr[i] = i < world ? reinterpret_cast<void*>(peer_ptrs[i] + off_bytes) : nullptr;
    q.ptr[i] = i < world ? reinterpret_cast<uint32_t*>(pad_ptrs[i]) : nullptr;
  }
}

cudaError_t symm_all_gather(const uint64_t* peer_ptrs, const uint64_t* pad_ptrs, size_t src_off_bytes, void* out,
                            size_t bytes, int rank, int world, int channel, uint32_t epoch, uint32_t* block_counter,
                            int num_sms, cudaStream_t stream) {
  if (world > kMaxWorld || bytes % 16 != 0 || channel >= kPadChannels) return cudaErrorInvalidValue;
  Peers p; Pads q;
  configure_kernels_once();
  fill(p, q, peer_ptrs, pad_ptrs, world, src_off_bytes);
  if (tma_min_bytes() > 0 && bytes >= (size_t)tma_min_bytes()) {
    static cudaError_t cfg = allow_smem(multi_copy_tma_kernel, copy_smem());
    if (cfg != cudaSuccess) return cfg;
    CopyList cl;
    for (int r = 0; r < kMaxWorld; ++r) {
      cl.src[r] = r < world ? (const uint8_t*)p.ptr[r] : nullptr;
      cl.dst[r] = r < world ? (uint8_t*)out + (size_t)r * bytes : nullptr;
    }
    const size_t chunks = (bytes + copy_chunk() - 1) / copy_chunk();
    const int grid = (int)(chunks < (size_t)tma_ctas() ? chunks : (size_t)tma_ctas());
    multi_copy_tma_kernel<<<grid, 32, copy_smem(), stream>>>(cl, q, bytes, rank, world, copy_chunk(), copy_stages(),
                                                             channel, epoch, block_counter);
    return cudaGetLastError();
  }
  all_gather_kernel<<<grid_for(bytes * world, num_sms), 512, 0, stream>>>(p, q, (uint8_t*)out, bytes, rank, world,
                                                                          channel, epoch, block_counter);
  return cudaGetLastError();
}

cudaError_t symm_reduce_scatter(const uint64_t* peer_ptrs, const uint64_t* pad_ptrs, size_t src_off_bytes, void* out,
                                size_t n, bool in_bf16, bool out_fp32, float scale, int rank, int world, int channel,
                                uint32_t epoch, uint32_t* block_counter, int num_sms, cudaStream_t stream) {
  if (world > kMaxWorld || channel >= kPadChannels) return cudaErrorInvalidValue;
  if (n % (in_bf16 ? 8 : 4) != 0) return cudaErrorInvalidValue;
  Peers p; Pads q;
  configure_kernels_once();
  fill(p, q, peer_ptrs, pad_ptrs, world, src_off_bytes);
  const size_t slice_bytes = n * (in_bf16 ? 2 : 4);
  if (tma_min_bytes() > 0 && slice_bytes >= (size_t)tma_min_bytes()) {
    uint32_t sub = (kTmaChunk / world) & ~1023u;          // one stage = `world` sub-chunks <= 32 KB
    const int stages = kTmaStages;
    const int smem = stages * (int)sub * world + 1024 + 256;
    const size_t chunks = (slice_bytes + sub - 1) / sub;
    const int grid = (int)(chunks < (size_t)rs_ctas() ? chunks : (size_t)rs_ctas());
#define TB_RS_TMA(IN, OUT)                                                                                         \
  do {                                                                                                             \
    static cudaError_t cfg = allow_smem(reduce_scatter_tma_kernel<IN, OUT>, kTmaSmem);                             \
    if (cfg != cudaSuccess) return cfg;                                                                            \
    reduce_scatter_tma_kernel<IN, OUT><<<grid, 288, smem, stream>>>(p, q, (OUT*)out, n, scale, rank, world, sub,    \
                                                                    stages, channel, epoch, block_counter);        \
  } while (0)
    if (in_bf16 && out_fp32) TB_RS_TMA(__nv_bfloat16, float);
    else if (in_bf16) TB_RS_TMA(__nv_bfloat16, __nv_bfloat16);
    else if (out_fp32) TB_RS_TMA(float, float);
    else TB_RS_TMA(float, __nv_bfloat16);
#undef TB_RS_TMA
    return cudaGetLastError();
  }
  const int grid = grid_for(n * (in_bf16 ? 2 : 4) * world, num_sms);
#define TB_RS(IN, OUT)                                                                                          \
  reduce_scatter_kernel<IN, OUT><<<grid, 512, 0, stream>>>(p, q, (OUT*)out, n, scale, rank, world, channel, epoch, \
                                                            block_counter)
  if (in_bf16 && out_fp32) TB_RS(__nv_bfloat16, float);
  else if (in_bf16) TB_RS(__nv_bfloat16, __nv_bfloat16);
  else if (out_fp32) TB_RS(float, float);
  else TB_RS(float, __nv_bfloat16);
#undef TB_RS
  return cudaGetLastError();
}

cudaError_t symm_all_to_all(const uint64_t* peer_ptrs, const uint64_t* pad_ptrs, size_t src_off_bytes, void* out,
                            size_t chunk_bytes, int rank, int world, int channel, uint32_t epoch,
                            uint32_t* block_counter, int num_sms, cudaStream_t stream) {
  if (world > kMaxWorld || chunk_bytes % 16 != 0 || channel >= kPadChannels) return cudaErrorInvalidValue;
  Peers p; Pads q;
  configure_kernels_once();
  fill(p, q, peer_ptrs, pad_ptrs, world, src_off_bytes);
  if (tma_min_bytes() > 0 && chunk_bytes >= (size_t)tma_min_bytes()) {
    static cudaError_t cfg = allow_smem(multi_copy_tma_kernel, copy_smem());
    if (cfg != cudaSuccess) return cfg;
    CopyList cl;
    for (int r = 0; r < kMaxWorld; ++r) {
      cl.src[r] = r < world ? (const uint8_t*)p.ptr[r] + (size_t)rank * chunk_bytes : nullptr;
      cl.dst[r] = r < world ? (uint8_t*)out + (size_t)r * chunk_bytes : nullptr;
    }
    const size_t chunks = (chunk_bytes + copy_chunk() - 1) / copy_chunk();
    const int grid = (int)(chunks < (size_t)tma_ctas() ? chunks : (size_t)tma_ctas());
    multi_copy_tma_kernel<<<grid, 32, copy_smem(), stream>>>(cl, q, chunk_bytes, rank, world, copy_chunk(),
                                                             copy_stages(), channel, epoch, block_counter);
    return cudaGetLastError();
  }
  all_to_all_kernel<<<grid_for(chunk_bytes * world, num_sms), 512, 0, stream>>>(p, q, (uint8_t*)out, chunk_bytes, rank,
                                                                                world, channel, epoch, block_counter);
  return cudaGetLastError();
}

// ---- IPC plumbing -----------------------------------------------------------------------------------------
cudaError_t symm_alloc(size_t bytes, void** ptr) {
  cudaError_t e = cudaMalloc(ptr, bytes);
  if (e != cudaSuccess) return e;
  return cudaMemset(*ptr, 0, bytes);
}
cudaError_t symm_free(void* ptr) { return cudaFree(ptr); }
cudaError_t symm_get_handle(void* ptr, void* handle64) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
  if (e != cudaSuccess) return e;
  memcpy(handle64, &h, sizeof(h));
  return cudaSuccess;
}
cudaError_t symm_open_handle(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  return cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
}
cudaError_t symm_close_handle(void* ptr) { return cudaIpcCloseMemHandle(ptr); }

}  // namespace tb
