// Collectives carried INSIDE compute kernels ("carry jobs").
//
// FSDP moves ~0.4 GB over NVLink per decoder layer and direction (parameter all-gather, gradient reduce-scatter).
// Run as stand-alone kernels on side streams those transfers fight the persistent wgmma GEMMs for SMs, L2 and issue
// slots.  Here the transfer is a
// ROLE of the GEMM kernel itself: warp 3 of every GEMM CTA (idle under static tile scheduling) is a copy engine that
// moves a slice of the pending collective with TMA bulk copies through a small private smem ring while warps 0 and 4-11
// run the wgmma pipeline of the same CTA.  No extra kernel, no extra stream, no SM taken from the GEMM, and the
// bytes per launch are budgeted from the GEMM's FLOPs so the transfer ends before the mainloop does.
//
//   kind 1  all-gather slice : peer shard r  --cp.async.bulk-->  smem  --cp.async.bulk-->  local gathered buffer
//   kind 2  reduce-scatter   : `world` peer slices --cp.async.bulk--> smem, summed in fp32 by the warp, scaled, written
//                              to the local gradient shard (fp32 or bf16, optionally accumulating), and the sum of
//                              squares of the result is accumulated for the global gradient norm (no separate pass)
//
// Cross-rank protocol (epoch e of a channel on the symmetric signal pad, see comm/symm_comm.cu for the layout):
//   entry : a rank publishes "my source buffer is final" (symm_signal, a one-warp kernel ordered after the producers
//           of the buffer) into slot [entry channel][rank] of every peer -- for gradients when a unit's backward ends,
//           for parameter shards ONCE per step after the optimizer; every slice waits until all peers have published
//           >= its entry epoch before touching peer memory.  The flag is tied to the point where the data becomes
//           final, not to the launch that happens to carry the first slice: ranks whose byte budgets differ never
//           wait on each other's scheduling, and a job may be enqueued later than its data is ready (slack against
//           GPUs that run a phase a few percent slower).
//   exit  : the LAST slice, once every CTA of this rank has finished, publishes e into slot [ch][8 + rank] of every
//           peer ("I am done reading your buffer") and does NOT wait; whoever is about to overwrite a source buffer
//           waits for those flags first (symm_wait_done, a one-warp kernel).
// Spins are bounded: after ~60 s without progress the kernel reports the stuck peer/channel/epoch and traps, so a lost
// rank surfaces as a CUDA error on the host instead of a silent hang.
//
// Reference parity: torchacc/dist/fsdp.py:196-230 (torch FSDP / XLA-FSDP all-gather + reduce-scatter per unit).
#pragma once
#include <stdio.h>

#include "../common/ptx.cuh"
#include "../common/spin.cuh"

namespace tb {

constexpr int kCarryMaxWorld = 8;
constexpr uint32_t kCarryStageBytes = 8192;
constexpr int kCarryStages = 3;
constexpr int kCarrySmemBytes = kCarryStages * (int)kCarryStageBytes + 64;   // ring + mbarriers
constexpr int kCarrySlots = 2;                                              // slices one launch can carry

struct CarrySlice {
  int kind;                               // 0 none, 1 all-gather copy, 2 reduce-scatter
  int rank, world;
  int channel;                            // exit ("done") flags: slot [channel][8 + rank] = epoch
  uint32_t epoch;
  int entry_channel;                      // entry ("source buffers are final") flags: slot [entry_channel][rank] >=
  uint32_t entry_epoch;                   //   entry_epoch on every rank before peer memory is touched
  int signal_entry, signal_exit;
  const uint8_t* src[kCarryMaxWorld];     // kind 1: peer r's shard; kind 2: peer r's flat buffer + rank * bytes
  uint8_t* dst;                           // kind 1: gathered buffer (shard r at dst + r * bytes); kind 2: output shard
  uint32_t* pads[kCarryMaxWorld];
  long long bytes;                        // per-source bytes of the whole job
  uint32_t chunk_bytes;                   // kind 1: bytes per chunk; kind 2: bytes per source per chunk
  uint32_t chunk_begin, chunk_end;        // this launch's part of the job's chunk space
  uint32_t* block_counter;
  float scale;                            // kind 2
  int in_bf16, out_fp32, accumulate;      // kind 2
  float* stats;                           // kind 2: [0] += sum of squares of the result, [1] = 1 if non-finite
};

struct CarryArgs {
  CarrySlice slice[kCarrySlots];
  // optional timing record of CTA 0 (tb_carry_set_debug): per launch 8 x u64 globaltimer ns
  //   [0] role start  [1] slice 0 entry passed  [2] slice 0 done  [3] slice 1 entry passed  [4] slice 1 done
  //   [5] chunks of slice 0 | chunks of slice 1 << 32   [6] kinds   [7] launch index
  unsigned long long* debug;
};

TB_DEVICE unsigned long long carry_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// One warp.  `ring` / `bars`: shared-memory addresses of kCarryStages x kCarryStageBytes bytes and kCarryStages
// mbarriers (initialised by the caller with count 1).  `it` is the ring position carried across slices of one launch.
TB_DEVICE void carry_run_slice(const CarrySlice& s, uint32_t ring, uint32_t bars, uint32_t& it, int cta, int num_ctas,
                                unsigned long long* dbg = nullptr) {
  const uint32_t lane = lane_id();
  constexpr uint32_t kSlotBase = 16;   // pad slots per channel: [0,8) entry, [8,16) exit
  // ---- entry ----
  if (s.signal_entry && cta == 0 && (int)lane < s.world) {
    __threadfence_system();
    carry_st_release_sys(s.pads[lane] + s.entry_channel * kSlotBase + s.rank, s.entry_epoch);
  }
  if ((int)lane < s.world)
    spin_until_epoch(s.pads[s.rank] + s.entry_channel * kSlotBase + lane, s.entry_epoch, s.rank, (int)lane,
                     s.entry_channel, "carry entry");
  __syncwarp();
  asm volatile("fence.proxy.async;" ::: "memory");   // peers' generic-proxy writes (acquired above) -> TMA reads
  if (dbg != nullptr && lane == 0) dbg[0] = carry_now_ns();

  const uint32_t n = s.chunk_end > s.chunk_begin ? s.chunk_end - s.chunk_begin : 0;
  const uint32_t mine = n > (uint32_t)cta ? (n - cta + num_ctas - 1) / num_ctas : 0;   // chunks begin+cta, +num_ctas...
  if (s.kind == 1) {
    if (lane == 0 && mine > 0) {
      const uint32_t cps = (uint32_t)((s.bytes + s.chunk_bytes - 1) / s.chunk_bytes);   // chunks per source shard
      auto locate = [&](uint32_t j, const uint8_t*& sp, uint8_t*& dp, uint32_t& len) {
        const uint32_t c = s.chunk_begin + cta + j * num_ctas;
        const int r = (s.rank + (int)(c / cps)) % s.world;      // own shard first (local copy), then the ring
        const long long off = (long long)(c % cps) * s.chunk_bytes;
        sp = s.src[r] + off;
        dp = s.dst + (long long)r * s.bytes + off;
        const long long left = s.bytes - off;
        len = left < (long long)s.chunk_bytes ? (uint32_t)left : s.chunk_bytes;
      };
      auto issue = [&](uint32_t j) {
        const uint8_t* sp; uint8_t* dp; uint32_t len;
        locate(j, sp, dp, len);
        const uint32_t st = (it + j) % kCarryStages;
        mbar_arrive_expect_tx(bars + 8u * st, len);
        bulk_load_hint(ring + st * kCarryStageBytes, sp, len, bars + 8u * st, kEvictFirst);
      };
      uint32_t issued = 0;
      for (; issued < (uint32_t)kCarryStages - 1 && issued < mine; ++issued) issue(issued);
      for (uint32_t i = 0; i < mine; ++i) {
        const uint32_t st = (it + i) % kCarryStages;
        mbar_wait_relaxed(bars + 8u * st, ((it + i) / kCarryStages) & 1);
        const uint8_t* sp; uint8_t* dp; uint32_t len;
        locate(i, sp, dp, len);
        bulk_store_hint(dp, ring + st * kCarryStageBytes, len, kEvictFirst);
        tma_store_commit();
        if (issued < mine) {
          tma_store_wait_read<1>();      // every store but the newest has left smem: stage (i-1) % stages is free
          issue(issued++);
        }
      }
      tma_store_wait<0>();               // landed in local memory before this kernel (and the stream) moves on
    }
    it += mine;
    __syncwarp();
  } else if (s.kind == 2) {
    const uint32_t sub = s.chunk_bytes;
    const uint32_t stage_stride = kCarryStageBytes;
    float sq = 0.f;
    auto issue = [&](uint32_t j) {       // lane 0 only
      const uint32_t c = s.chunk_begin + cta + j * num_ctas;
      const long long off = (long long)c * sub;
      const long long left = s.bytes - off;
      const uint32_t len = left < (long long)sub ? (uint32_t)left : sub;
      const uint32_t st = (it + j) % kCarryStages;
      mbar_arrive_expect_tx(bars + 8u * st, len * s.world);
      for (int p = 0; p < s.world; ++p) {
        const int r = (s.rank + p) % s.world;
        bulk_load_hint(ring + st * stage_stride + p * sub, s.src[r] + off, len, bars + 8u * st, kEvictFirst);
      }
    };
    uint32_t issued = 0;
    if (lane == 0)
      for (; issued < (uint32_t)kCarryStages - 1 && issued < mine; ++issued) issue(issued);
    issued = __shfl_sync(0xffffffffu, issued, 0);
    for (uint32_t i = 0; i < mine; ++i) {
      const uint32_t st = (it + i) % kCarryStages;
      if (lane == 0) mbar_wait_relaxed(bars + 8u * st, ((it + i) / kCarryStages) & 1);
      __syncwarp();                       // lane 0 observed the phase; the warp barrier orders the smem reads below
      const uint32_t c = s.chunk_begin + cta + i * num_ctas;
      const long long off = (long long)c * sub;
      const long long left = s.bytes - off;
      const uint32_t len = left < (long long)sub ? (uint32_t)left : sub;
      const uint32_t sbase = ring + st * stage_stride;
      if (s.in_bf16) {
        const uint32_t nvec = len >> 4;                                  // 8 bf16 per 16-byte vector
        const long long e0 = off >> 1;                                   // first output element of this chunk
        for (uint32_t v = lane; v < nvec; v += 32) {
          float acc[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = 0.f;
          for (int p = 0; p < s.world; ++p) {
            uint4 u;
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                         : "r"(sbase + p * sub + v * 16));
            float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c2 = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
            acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
            acc[4] += c2.x; acc[5] += c2.y; acc[6] += d.x; acc[7] += d.y;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] *= s.scale;
          if (s.out_fp32) {
            float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(s.dst) + e0 + (long long)v * 8);
            if (s.accumulate) {
              const float4 o0 = op[0], o1 = op[1];
              acc[0] += o0.x; acc[1] += o0.y; acc[2] += o0.z; acc[3] += o0.w;
              acc[4] += o1.x; acc[5] += o1.y; acc[6] += o1.z; acc[7] += o1.w;
            }
            __stcs(op, make_float4(acc[0], acc[1], acc[2], acc[3]));          // streaming: read once by the optimizer
            __stcs(op + 1, make_float4(acc[4], acc[5], acc[6], acc[7]));
          } else {
            uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(s.dst) + e0 + (long long)v * 8);
            if (s.accumulate) {
              const uint4 o = *op;
              float2 a = unpack_bf16x2(o.x), b = unpack_bf16x2(o.y), c2 = unpack_bf16x2(o.z), d = unpack_bf16x2(o.w);
              acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
              acc[4] += c2.x; acc[5] += c2.y; acc[6] += d.x; acc[7] += d.y;
            }
            uint4 o;
            o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
            o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
            *op = o;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) sq += acc[j] * acc[j];
        }
      } else {
        const uint32_t nvec = len >> 4;                                  // 4 fp32 per vector
        const long long e0 = off >> 2;
        for (uint32_t v = lane; v < nvec; v += 32) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
          for (int p = 0; p < s.world; ++p) {
            uint4 u;
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                         : "r"(sbase + p * sub + v * 16));
            acc[0] += __uint_as_float(u.x); acc[1] += __uint_as_float(u.y);
            acc[2] += __uint_as_float(u.z); acc[3] += __uint_as_float(u.w);
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j] *= s.scale;
          if (s.out_fp32) {
            float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(s.dst) + e0 + (long long)v * 4);
            if (s.accumulate) {
              const float4 o0 = *op;
              acc[0] += o0.x; acc[1] += o0.y; acc[2] += o0.z; acc[3] += o0.w;
            }
            *op = make_float4(acc[0], acc[1], acc[2], acc[3]);
          } else {
            uint2* op = reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(s.dst) + e0 + (long long)v * 4);
            if (s.accumulate) {
              const uint2 o = *op;
              float2 a = unpack_bf16x2(o.x), b = unpack_bf16x2(o.y);
              acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
            }
            uint2 o;
            o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
            *op = o;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) sq += acc[j] * acc[j];
        }
      }
      __syncwarp();                       // every lane has finished reading this stage
      if (lane == 0 && issued < mine) {
        fence_proxy_async_smem();         // our generic-proxy reads precede the next asynchronous write of the stage
        issue(issued);
      }
      if (issued < mine) ++issued;
    }
    it += mine;
    if (s.stats != nullptr) {
      sq = warp_reduce_sum(sq);
      if (lane == 0 && mine > 0) {
        atomicAdd(s.stats, sq);
        if (!(fabsf(sq) <= 3.0e38f)) atomicExch(s.stats + 1, 1.0f);     // inf / nan
      }
    }
    __syncwarp();
  }
  if (dbg != nullptr && lane == 0) dbg[1] = carry_now_ns();
  // ---- exit ----
  if (s.signal_exit) {
    uint32_t last = 0;
    if (lane == 0) {
      __threadfence();
      last = (atomicAdd(s.block_counter, 1u) == (uint32_t)num_ctas - 1) ? 1u : 0u;
      if (last) *s.block_counter = 0;     // re-arm (the next user of this counter is stream-ordered after us)
    }
    last = __shfl_sync(0xffffffffu, last, 0);
    if (last && (int)lane < s.world) {
      __threadfence_system();
      carry_st_release_sys(s.pads[lane] + s.channel * kSlotBase + 8 + s.rank, s.epoch);
    }
    __syncwarp();
  }
}

// All slices of one launch.  Called by a full warp; initialises its own mbarriers.
TB_DEVICE void carry_role(const CarryArgs& ca, uint32_t ring, uint32_t bars, int cta, int num_ctas) {
  if (lane_id() == 0) {
    for (int s = 0; s < kCarryStages; ++s) mbar_init(bars + 8u * s, 1);
    fence_mbar_init();
  }
  __syncwarp();
  uint32_t it = 0;
  unsigned long long* dbg = (ca.debug != nullptr && cta == 0) ? ca.debug : nullptr;
  if (dbg != nullptr && lane_id() == 0) {
    dbg[0] = carry_now_ns();
    dbg[5] = (unsigned long long)(ca.slice[0].chunk_end - ca.slice[0].chunk_begin) |
             ((unsigned long long)(ca.slice[1].chunk_end - ca.slice[1].chunk_begin) << 32);
    dbg[6] = (unsigned long long)ca.slice[0].kind | ((unsigned long long)ca.slice[1].kind << 8);
  }
#pragma unroll 1
  for (int i = 0; i < kCarrySlots; ++i)
    if (ca.slice[i].kind != 0)
      carry_run_slice(ca.slice[i], ring, bars, it, cta, num_ctas, dbg != nullptr ? dbg + 1 + 2 * i : nullptr);
}

}  // namespace tb
