"""Fused tensor-parallel kernels vs the unfused baseline (NCCL collective + GEMM), Llama-3-8B TP shapes.

    torchrun --nproc-per-node N benchmarks/fused_tp_bench.py [--tokens 8192]

Per op: device time (CUDA events, L2 flushed between iterations, max over ranks) of
  fused   : one kernel (all-gather->GEMM) / GEMM with peer-store epilogue + reduce kernel (GEMM->reduce-scatter)
  unfused : NCCL all_gather_into_tensor / reduce_scatter_tensor + the same wgmma GEMM
  gemm    : the GEMM alone (lower bound: perfect overlap)
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timeit(fn, iters, flush):
    ts = []
    for i in range(iters + 3):
        flush.zero_()
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= 3:
            ts.append(a.elapsed_time(b))
    t = torch.tensor(sorted(ts)[len(ts) // 2], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    rank = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    world = dist.get_world_size()
    dev = torch.device("cuda", rank)
    from torchacc_b200.ops.linear import gemm
    from torchacc_b200.parallel.fused_tp import make_fused_tp
    f = make_fused_tp(dist.group.WORLD, dev)
    assert f is not None, "fused TP kernels unavailable"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    T, H, QKV, FF = args.tokens, 4096, 6144, 14336
    rows = T // world
    res = []
    torch.manual_seed(rank)
    # ---- all-gather -> GEMM (column-parallel: qkv_proj, gate_up_proj) ----
    for name, N in (("qkv_proj", QKV // world), ("gate_up_proj", 2 * FF // world)):
        x = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, H, device=dev, dtype=torch.bfloat16) * 0.02
        full = torch.empty(T, H, device=dev, dtype=torch.bfloat16)
        y = torch.empty(T, N, device=dev, dtype=torch.bfloat16)

        def unfused():
            dist.all_gather_into_tensor(full, x)
            gemm(full, w, out=y)
        t_f = timeit(lambda: f.ag_gemm(x, w), args.iters, flush)
        t_u = timeit(unfused, args.iters, flush)
        t_g = timeit(lambda: gemm(full, w, out=y), args.iters, flush)
        yf, _ = f.ag_gemm(x, w)
        unfused()
        err = float((yf.float() - y.float()).abs().max())
        res.append(dict(op="ag_gemm", layer=name, M=T, N=N, K=H, fused_ms=t_f, unfused_ms=t_u, gemm_only_ms=t_g,
                        speedup=t_u / t_f, tflops_fused=2.0 * T * N * H / t_f / 1e9, max_abs_err=err))
    # ---- GEMM -> reduce-scatter (row-parallel: o_proj, down_proj) ----
    for name, K in (("o_proj", H // world), ("down_proj", FF // world)):
        x = torch.randn(T, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(H, K, device=dev, dtype=torch.bfloat16) * 0.02
        part = torch.empty(T, H, device=dev, dtype=torch.bfloat16)
        out = torch.empty(rows, H, device=dev, dtype=torch.bfloat16)

        def unfused():
            gemm(x, w, out=part)
            dist.reduce_scatter_tensor(out, part)
        t_f = timeit(lambda: f.gemm_rs(x, w), args.iters, flush)
        t_u = timeit(unfused, args.iters, flush)
        t_g = timeit(lambda: gemm(x, w, out=part), args.iters, flush)
        of = f.gemm_rs(x, w)
        unfused()
        err = float((of.float() - out.float()).abs().max())
        res.append(dict(op="gemm_rs", layer=name, M=T, N=H, K=K, fused_ms=t_f, unfused_ms=t_u, gemm_only_ms=t_g,
                        speedup=t_u / t_f, tflops_fused=2.0 * T * H * K / t_f / 1e9, max_abs_err=err))
    # roofline per the profiling recipe: target time = the slower of FLOPs / GEMM peak and the bytes that must
    # cross NVLink / link bandwidth (H100 SXM data sheet: 989 TFLOP/s dense bf16, 450 GB/s per direction per GPU;
    # MEASURED_PEAKS.json, when present, replaces the compute figure with a measured one)
    peak_tf, link_gbs = 989.0, 450.0
    try:
        mp = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
        peak_tf = float(mp.get("bf16_tflops", peak_tf))
    except Exception:
        pass
    for r in res:
        flops = 2.0 * r["M"] * r["N"] * r["K"]
        if r["op"] == "ag_gemm":      # remote rows of the gathered activation
            nv_bytes = r["M"] * r["K"] * 2 * (world - 1) / world
        else:                          # partial output tiles pushed to their owners
            nv_bytes = r["M"] * r["N"] * 2 * (world - 1) / world
        t_c, t_n = flops / (peak_tf * 1e12) * 1e3, nv_bytes / (link_gbs * 1e9) * 1e3
        r["roofline_ms"] = max(t_c, t_n)
        r["roofline_bound"] = "compute" if t_c >= t_n else "nvlink"
        r["roofline_frac_fused"] = r["roofline_ms"] / r["fused_ms"]
        r["roofline_frac_unfused"] = r["roofline_ms"] / r["unfused_ms"]
    if dist.get_rank() == 0:
        for r in res:
            print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()} | {"world": world}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
