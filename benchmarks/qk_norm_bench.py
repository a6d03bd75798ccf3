"""The fused per-head QK-RMSNorm + RoPE kernels (csrc/ops/norm_rope_act.cu) at the Qwen3-8B layer shape, T = 8192
tokens (2 x 4096), Hq = 32, Hk = 8, D = 128, bf16, against the composition of existing kernels they replace: contiguous
copies of the q and k columns, ``rmsnorm`` on each, the normalised q / k packed back next to v, and ``rope_qkv_``.

Forward and backward are timed with CUDA events over --iters calls after --warmup, fused and composed alternating in
one process (median of --reps windows each).  The backward is timed by re-running autograd on one retained graph.
GB/s counts the bytes the fused kernels must move (forward: read qkv, write out and rstd; backward: read g, the q / k
columns of qkv and rstd, write dqkv), and is also given as a share of the H100 SXM's 3.35 TB/s.  Prints one JSON
line with the card's name and power limit.

    python benchmarks/qk_norm_bench.py [--T 8192] [--hq 32] [--hk 8] [--D 128] [--iters 50] [--warmup 10] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        limit = "unknown"
    return name, limit


def time_alternating(fns, iters, warmup, reps):
    """Median ms per call of each function, the timing windows of the functions interleaved."""
    for fn in fns:
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    out = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            out[i].append(a.elapsed_time(b) / iters)
    return [statistics.median(o) for o in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=8192)
    ap.add_argument("--hq", type=int, default=32)
    ap.add_argument("--hk", type=int, default=8)
    ap.add_argument("--D", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qk_norm_bench needs a CUDA device")
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import qk_norm_rope_qkv, rmsnorm, rope_qkv_, rope_tables
    nat.require()
    T, hq, hk, D = args.T, args.hq, args.hk, args.D
    seq_len, eps = 4096, 1e-6
    dev = "cuda"
    torch.manual_seed(0)
    cos, sin = rope_tables(40960, D, 1e6, device=dev)
    qkv = torch.randn(T, (hq + 2 * hk) * D, device=dev).bfloat16().requires_grad_()
    wq = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16().requires_grad_()
    wk = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16().requires_grad_()
    g = torch.randn(T, (hq + 2 * hk) * D, device=dev).bfloat16()

    def fused():
        return qk_norm_rope_qkv(qkv, hq, hk, D, wq, wk, eps, cos, sin, None, seq_len)

    def composed():
        q = qkv[:, :hq * D].contiguous().view(T * hq, D)
        k = qkv[:, hq * D:(hq + hk) * D].contiguous().view(T * hk, D)
        qn, _ = rmsnorm(q, wq, eps)
        kn, _ = rmsnorm(k, wk, eps)
        packed = torch.cat([qn.view(T, hq * D), kn.view(T, hk * D), qkv[:, (hq + hk) * D:]], 1)
        return rope_qkv_(packed, hq, hk, D, cos, sin, None, seq_len)

    def fwd(fn):
        def run():
            with torch.no_grad():
                fn()
        return run

    def bwd(fn):
        out = fn()

        def run():
            torch.autograd.grad(out, (qkv, wq, wk), g, retain_graph=True)
        return run

    # the two paths agree (one bf16 rounding apart: the composition rounds z before the rotation)
    diff = float((fused() - composed()).float().abs().max())
    f_fused, f_comp = time_alternating([fwd(fused), fwd(composed)], args.iters, args.warmup, args.reps)
    b_fused, b_comp = time_alternating([bwd(fused), bwd(composed)], args.iters, args.warmup, args.reps)
    e = 2                                                                # bytes per bf16 element
    all_el, qk_el, rows = T * (hq + 2 * hk) * D, T * (hq + hk) * D, T * (hq + hk)
    fwd_bytes = 2 * all_el * e + rows * 4
    bwd_bytes = (2 * all_el + qk_el) * e + rows * 4
    name, limit = card()
    res = {"bench": "qk_norm_rope", "T": T, "hq": hq, "hk": hk, "D": D, "gpu": name, "power_limit": limit,
           "max_abs_diff_vs_composition": diff, "fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes}
    for tag, ms, nbytes in (("fwd_fused", f_fused, fwd_bytes), ("fwd_composed", f_comp, fwd_bytes),
                            ("bwd_fused", b_fused, bwd_bytes), ("bwd_composed", b_comp, bwd_bytes)):
        gbps = nbytes / ms / 1e6
        res[tag + "_ms"] = round(ms, 4)
        res[tag + "_GBps"] = round(gbps, 1)
        res[tag + "_of_3.35TBps"] = round(gbps * 1e9 / HBM_BYTES_PER_S, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
