// Thin inline-PTX layer for sm_90a: mbarrier, TMA, cluster helpers (the warpgroup MMA wrappers are in wgmma.cuh).
// Everything here is a direct wrapper of one PTX instruction so kernels read like the
// hardware protocol they implement.  Compile with -gencode arch=compute_90a,code=sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace tb {

#define TB_DEVICE __device__ __forceinline__

// ----------------------------------------------------------------------------------------------
// Generic helpers
// ----------------------------------------------------------------------------------------------
TB_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

TB_DEVICE uint32_t lane_id() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(r));
  return r;
}

TB_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

TB_DEVICE bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .b32 %%rx;\n\t"
      ".reg .pred %%px;\n\t"
      "elect.sync %%rx|%%px, %1;\n\t"
      "@%%px mov.s32 %0, 1;\n\t"
      "}\n"
      : "+r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}

// Named barrier `id` (1..15; 0 is __syncthreads) over `count` threads, a multiple of 32.
TB_DEVICE void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
TB_DEVICE void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
TB_DEVICE uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
TB_DEVICE void st_shared_v2_f32(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

TB_DEVICE void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
TB_DEVICE void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
TB_DEVICE void cluster_sync() {
  cluster_arrive();
  cluster_wait();
}

// Map a local shared-memory address to the same offset in CTA `rank` of the cluster.
TB_DEVICE uint32_t mapa_shared(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
TB_DEVICE void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
TB_DEVICE void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
TB_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

TB_DEVICE void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Arrive on a barrier living in another CTA of the cluster (address from mapa_shared).
TB_DEVICE void mbar_arrive_cluster(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
TB_DEVICE void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
TB_DEVICE void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
TB_DEVICE bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
TB_DEVICE void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// Low-duty wait for side roles (copy engines): back off between polls so the spinning warp does not compete with the
// MMA warps of the same SM sub-partition for issue slots (and power) while a transfer is in flight.
TB_DEVICE void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(128);
}
// Cluster-scope acquire variant: needed when the arrival came from the peer CTA.
TB_DEVICE bool mbar_try_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
TB_DEVICE void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait_cluster(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ----------------------------------------------------------------------------------------------
TB_DEVICE void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}

// L2 cache-hint policies (same encodings CUTLASS uses for CacheHintSm90).
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

TB_DEVICE void tma_load_2d(uint32_t smem_dst, const void* desc, uint32_t bar, int32_t c0, int32_t c1,
                           uint64_t hint = kEvictNormal) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}
TB_DEVICE void tma_load_3d(uint32_t smem_dst, const void* desc, uint32_t bar, int32_t c0, int32_t c1, int32_t c2,
                           uint64_t hint = kEvictNormal) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(hint)
      : "memory");
}
TB_DEVICE void tma_load_4d(uint32_t smem_dst, const void* desc, uint32_t bar, int32_t c0, int32_t c1, int32_t c2,
                           int32_t c3, uint64_t hint = kEvictNormal) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "l"(hint)
      : "memory");
}
TB_DEVICE void tma_store_2d(const void* desc, uint32_t smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
TB_DEVICE void tma_store_4d(const void* desc, uint32_t smem_src, int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
TB_DEVICE void tma_reduce_add_2d(const void* desc, uint32_t smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
TB_DEVICE void tma_reduce_add_3d(const void* desc, uint32_t smem_src, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// non-tensor bulk copies (contiguous bytes; 16-byte aligned, size % 16 == 0).  Source / destination may be any
// global address, including a peer GPU's memory mapped over NVLink.
TB_DEVICE void bulk_load(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar)
               : "memory");
}
TB_DEVICE void bulk_store(void* gdst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_src), "r"(bytes)
               : "memory");
}
// Same with an L2 cache policy (createpolicy / kEvict* constants): streaming traffic of the collectives must not evict
// the operand tiles the GEMMs keep L2-resident.
TB_DEVICE void bulk_load_hint(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}
TB_DEVICE void bulk_store_hint(void* gdst, uint32_t smem_src, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gdst),
               "r"(smem_src), "r"(bytes), "l"(policy)
               : "memory");
}
TB_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
TB_DEVICE void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
TB_DEVICE void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// Register reallocation between the warpgroups of a CTA (producer warps give registers to the MMA warpgroups)
// ----------------------------------------------------------------------------------------------
template <int N>
TB_DEVICE void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
TB_DEVICE void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// 4 x 4 transpose of 32-bit values inside each quad of lanes: afterwards x[s] of lane t holds what lane s had in x[t].
// Turns the 4-byte pieces of an MMA accumulator row into 16 contiguous bytes per lane.
TB_DEVICE void quad_transpose(uint32_t (&x)[4], uint32_t lane) {
#pragma unroll
  for (int m = 1; m <= 2; m <<= 1) {
    const bool up = (lane & m) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i & m) continue;
      const uint32_t send = up ? x[i] : x[i | m];
      const uint32_t got = __shfl_xor_sync(0xffffffffu, send, m);
      if (up) x[i] = got; else x[i | m] = got;
    }
  }
}

// Stores 8 consecutive 16-bit values (packed in pairs) of one row: one 16-byte store when alignment allows it.
TB_DEVICE void store_row8(uint16_t* dst, const uint32_t (&x)[4], int cols_left, bool vec_ok) {
  if (cols_left >= 8 && vec_ok) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(x[0], x[1], x[2], x[3]);
  } else {
    for (int j = 0; j < 8 && j < cols_left; ++j) dst[j] = (uint16_t)(x[j >> 1] >> (16 * (j & 1)));
  }
}

// ----------------------------------------------------------------------------------------------
// Small numeric helpers
// ----------------------------------------------------------------------------------------------
TB_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
TB_DEVICE float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
TB_DEVICE uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
TB_DEVICE float2 unpack_f16x2(uint32_t u) {
  __half2 v = *reinterpret_cast<__half2*>(&u);
  return __half22float2(v);
}
// 16-bit float pair in the kernel's element type (bf16 or fp16)
template <bool kBf16>
TB_DEVICE uint32_t pack_h2(float lo, float hi) {
  if constexpr (kBf16) return pack_bf16x2(lo, hi);
  else return pack_f16x2(lo, hi);
}
template <bool kBf16>
TB_DEVICE float2 unpack_h2(uint32_t u) {
  if constexpr (kBf16) return unpack_bf16x2(u);
  else return unpack_f16x2(u);
}
TB_DEVICE float fast_exp2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid(x) = 1 / (1 + 2^(-x log2 e)) with MUFU ex2 and rcp: a few fp32 ulps of relative error over the whole range,
// also for x << 0 where sigmoid(x) itself is tiny.  (0.5 + 0.5 tanh.approx(x / 2) is one MUFU op, but tanh.approx has
// about 2^-11 relative error, which near tanh = -1 is an absolute sigmoid error larger than sigmoid(x) for x < -8.)
// Large negative x: 2^(-x log2 e) overflows to +inf and the reciprocal gives 0.
TB_DEVICE float fast_sigmoid(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return r;
}

template <typename T>
TB_DEVICE T warp_reduce_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T>
TB_DEVICE T warp_reduce_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace tb
