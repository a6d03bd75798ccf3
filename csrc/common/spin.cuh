// Bounded device-side spins on cross-GPU flags (SURVEY 5.3: the reference has no failure detection).
// A wait that makes no progress for ~60 s prints which rank / channel / epoch it was waiting for and traps: the host sees a
// CUDA error instead of a hung GPU.
#pragma once
#include <stdio.h>

#include "ptx.cuh"

namespace tb {

TB_DEVICE void carry_st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
TB_DEVICE uint32_t carry_ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

constexpr long long kSpinTimeoutCycles = 120000000000ll;   // ~60 s at 1.9 GHz

// Wait until *flag (epoch numbering, wrap-safe) reaches `epoch`; trap with a diagnostic after kSpinTimeoutCycles.
TB_DEVICE void spin_until_epoch(const uint32_t* flag, uint32_t epoch, int my_rank, int peer, int channel,
                                const char* what) {
  if ((int32_t)(carry_ld_acquire_sys(flag) - epoch) >= 0) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while ((int32_t)(carry_ld_acquire_sys(flag) - epoch) < 0) {
    __nanosleep(64);
    if ((++polls & 0x3FFu) == 0 && clock64() - t0 > kSpinTimeoutCycles) {
      printf("[torchacc_b200] rank %d: timed out waiting for rank %d (%s, channel %d, epoch %u, flag %u)\n", my_rank,
             peer, what, channel, epoch, *(volatile const uint32_t*)flag);
      __trap();
    }
  }
}


// Plain counter variant (flags that count arrivals instead of carrying an epoch).
TB_DEVICE void spin_until_count(const uint32_t* flag, uint32_t target, int my_rank, int peer, const char* what) {
  spin_until_epoch(flag, target, my_rank, peer, -1, what);
}

}  // namespace tb
