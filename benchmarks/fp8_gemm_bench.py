#!/usr/bin/env python
"""MX-FP8 vs bf16 wgmma GEMM on the four Llama-3-8B linear shapes (T = 8192 tokens), plus the quantiser cost.
CUDA-event timing, 20 iterations after 5 warm-up runs, operands rotated over > 50 MB so L2 does not hold them."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torchacc_b200.ops import fp8  # noqa: E402
from torchacc_b200.ops.linear import gemm  # noqa: E402


def timeit(fn, n=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    dev = torch.device("cuda", 0)
    T = 8192
    shapes = [("qkv", T, 6144, 4096), ("o", T, 4096, 4096), ("gate_up", T, 28672, 4096), ("down", T, 4096, 14336)]
    rows = []
    for name, M, N, K in shapes:
        reps = max(2, int(300e6 // ((M + N) * K * 2)) + 1)          # rotate operand sets: > 50 MB (the L2 size) touched
        A = [(torch.randn(M, K, device=dev) * 0.5).bfloat16() for _ in range(reps)]
        B = [(torch.randn(N, K, device=dev) * 0.05).bfloat16() for _ in range(reps)]
        out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        i = [0]

        def bf():
            i[0] += 1
            gemm(A[i[0] % reps], B[i[0] % reps], out=out)
        Aq = [fp8.quantize_mxfp8(a)[0] for a in A]
        Bq = [fp8.quantize_mxfp8(b)[0] for b in B]

        def f8():
            i[0] += 1
            fp8.gemm_mxfp8(Aq[i[0] % reps], Bq[i[0] % reps], out=out)

        def qa():
            fp8.quantize_mxfp8(A[0], True, True)
        t_bf, t_f8, t_q = timeit(bf), timeit(f8), timeit(qa)
        fl = 2.0 * M * N * K
        rows.append({"shape": name, "M": M, "N": N, "K": K, "bf16_ms": round(t_bf, 4), "mxfp8_ms": round(t_f8, 4),
                     "speedup": round(t_bf / t_f8, 3), "bf16_tflops": round(fl / t_bf / 1e9, 1),
                     "mxfp8_tflops": round(fl / t_f8 / 1e9, 1), "quant_x_both_ms": round(t_q, 4)})
        print(json.dumps(rows[-1]), flush=True)


if __name__ == "__main__":
    main()
