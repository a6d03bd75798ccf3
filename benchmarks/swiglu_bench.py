"""The SwiGLU kernels (csrc/ops/norm_rope_act.cu) at the flagship MLP shape, T = 8192 tokens, F = 14336, bf16:
forward h = silu(g) u and backward (dg, du), on the fused gate|up layout [T, 2F].

Both kernels are meant to be HBM-bound; the sigmoid's MUFU work must stay hidden under the memory traffic.  Times
come from CUDA events over --iters launches after --warmup (median of --reps windows); GB/s counts the bytes each
kernel must move (forward: read g, u, write h; backward: read dh, g, u, write dg, du).  Prints one JSON line with the
card's name and power limit.  ``TORCHACC_B200_NATIVE_LIB`` selects the native library, so two builds can be compared
by alternating runs.

    python benchmarks/swiglu_bench.py [--T 8192] [--F 14336] [--iters 50] [--warmup 10] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        limit = "unknown"
    return name, limit


def time_ms(fn, iters, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=8192)
    ap.add_argument("--F", type=int, default=14336)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("swiglu_bench needs a CUDA device")
    from torchacc_b200 import _native as nat
    L = nat.require()
    T, F = args.T, args.F
    torch.manual_seed(0)
    gu = (torch.randn(T, 2 * F, device="cuda") * 3).bfloat16()
    dh = torch.randn(T, F, device="cuda").bfloat16()
    h = torch.empty(T, F, device="cuda", dtype=torch.bfloat16)
    dgu = torch.empty_like(gu)
    g_ptr, u_ptr = gu.data_ptr(), gu.data_ptr() + 2 * F

    def fwd():
        nat.check(L.tb_swiglu_fwd(g_ptr, u_ptr, h.data_ptr(), T, F, 2 * F, 2 * F, nat.num_sms(), nat.stream(), 1),
                  "tb_swiglu_fwd")

    def bwd():
        nat.check(L.tb_swiglu_bwd(dh.data_ptr(), g_ptr, u_ptr, dgu.data_ptr(), dgu.data_ptr() + 2 * F, T, F, 2 * F,
                                  2 * F, 2 * F, 2 * F, nat.num_sms(), nat.stream(), 1), "tb_swiglu_bwd")

    t_f = time_ms(fwd, args.iters, args.warmup, args.reps)
    t_b = time_ms(bwd, args.iters, args.warmup, args.reps)
    e = T * F * 2                                    # bytes of one [T, F] bf16 tensor
    name, limit = card()
    print(json.dumps({"bench": "swiglu", "T": T, "F": F, "lib": str(nat._SO), "gpu": name, "power_limit": limit,
                      "fwd_ms": round(t_f, 4), "fwd_GBps": round(3 * e / t_f / 1e6, 1),
                      "bwd_ms": round(t_b, 4), "bwd_GBps": round(5 * e / t_b / 1e6, 1)}))


if __name__ == "__main__":
    main()
