// Attention masking shared by the query-stationary kernels (flash_fwd.cu and the dQ kernel of flash_bwd.cu): the
// visible key range of a query row and the per-tile mask / ALiBi pass over a score accumulator.
// Causal is bottom-right aligned: query row i of a sequence sits at key position i + (k_len - q_len).
#pragma once
#include <math.h>
#include <stdint.h>

namespace tb {

// visible key range [lo, hi] for query row `row` (0-based inside its sequence)
__device__ __forceinline__ void key_bounds(int row, int q_len, int k_len, int causal, int wl, int wr, int& lo, int& hi) {
  const int pos = row + (k_len - q_len);
  int r = wr;
  if (causal) r = (wr < 0) ? 0 : min(wr, 0);
  hi = (r < 0) ? (k_len - 1) : min(k_len - 1, pos + r);
  lo = (wl < 0) ? 0 : max(0, pos - wl);
}

// Key tiles [j_lo, j_lo + n_tiles) of width `tile` that query rows [m0, m0 + rows) can see (n_tiles <= 0: none).
__device__ __forceinline__ void key_tile_range(int m0, int rows, int q_len, int k_len, int causal, int wl, int wr,
                                               int tile, int& j_lo, int& n_tiles) {
  int lo_first, hi_first, lo_last, hi_last;
  const int last_row = min(m0 + rows, q_len) - 1;
  key_bounds(m0, q_len, k_len, causal, wl, wr, lo_first, hi_first);
  key_bounds(last_row, q_len, k_len, causal, wl, wr, lo_last, hi_last);
  const int kmin = lo_first, kmax = hi_last;
  j_lo = kmin / tile;
  const int j_hi = (kmax < 0 || kmax < kmin) ? j_lo : (kmax / tile + 1);
  n_tiles = j_hi - j_lo;
}

// Mask / ALiBi pass over one m64nN score tile S = Q K^T in the wgmma accumulator layout: this thread holds rows r, r + 8
// (visible keys lo[i]..hi[i], key position pos_q[i]) and keys n0 + 8j + 2 quad + {0, 1} along the registers.
// Invisible entries become -inf.  With ALiBi the scores are scaled here and the bias -slope * |pos - key| is folded in
// (log2 units), so the caller continues with scale 1.  Interior tiles (every row of the warp sees every key, no ALiBi)
// skip the pass.
template <int N>
__device__ __forceinline__ void mask_score_tile(float (&s)[N / 2], int n0, uint32_t quad, const int (&lo)[2],
                                                const int (&hi)[2], const int (&pos_q)[2], bool has_alibi,
                                                float scale_log2, float slope_l2) {
  const bool interior = !has_alibi && n0 >= lo[0] && n0 >= lo[1] && n0 + N - 1 <= hi[0] && n0 + N - 1 <= hi[1];
  if (!__all_sync(0xffffffffu, interior)) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = e >> 1;
        const int kidx = n0 + 8 * j + 2 * (int)quad + (e & 1);
        float v = s[4 * j + e];
        if (has_alibi) v = fmaf(v, scale_log2, -slope_l2 * fabsf((float)(pos_q[i] - kidx)));
        s[4 * j + e] = (kidx >= lo[i] && kidx <= hi[i]) ? v : -INFINITY;
      }
  }
}

}  // namespace tb
