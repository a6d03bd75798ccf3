"""Attention micro-benchmark: our wgmma kernels vs the library paths (torch SDPA / flash-attn 2) on the Llama-3-8B
attention shape.  CUDA-event timing, L2 flushed between iterations.  ``--deterministic`` also times the deterministic
backward (atomic-free dQ kernel) in the same run; the card name and power limit are reported with the numbers."""
import argparse
import json
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timeit(fn, iters=10, warmup=3):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    ts = []
    for i in range(iters):
        flush.fill_(i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts), sum(ts) / len(ts)


def device_desc():
    """Card name and power limit (W) of cuda:0, read with nvidia-smi when it is available."""
    desc = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        desc["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        desc["power_limit_w"] = None
    return desc


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=2)
    p.add_argument("--seq", type=int, default=4096)
    p.add_argument("--hq", type=int, default=32)
    p.add_argument("--hk", type=int, default=8)
    p.add_argument("--d", type=int, default=128)
    p.add_argument("--only", default="", help="native: skip the library paths")
    p.add_argument("--deterministic", action="store_true",
                   help="also time the native deterministic backward (deterministic=True)")
    a = p.parse_args()
    from torchacc_b200.ops import attention as A
    B, S, Hq, Hk, D = a.batch, a.seq, a.hq, a.hk, a.d
    dev = "cuda"
    q = torch.randn(B, S, Hq, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(B, S, Hk, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(B, S, Hk, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(B, S, Hq, D, device=dev, dtype=torch.bfloat16)
    fwd_flops = 4 * B * S * S * Hq * D * 0.5
    res = {}

    def bench(name, fwd):
        out = fwd()
        t_f = timeit(fwd)
        def fb():
            o = fwd()
            o.backward(do)
        t_fb = timeit(fb)
        bwd = t_fb[0] - t_f[0]
        res[name] = {"fwd_ms": t_f[0], "fwd_tflops": fwd_flops / t_f[0] * 1e-9, "bwd_ms": bwd,
                     "bwd_tflops": 2.5 * fwd_flops / bwd * 1e-9}
        print(name, json.dumps(res[name]), flush=True)

    A.set_attention_backend("native")
    bench("tb_native", lambda: A.flash_attn_func(q, k, v, causal=True))
    if a.deterministic:
        bench("tb_native_deterministic", lambda: A.flash_attn_func(q, k, v, causal=True, deterministic=True))
    dev_desc = device_desc()
    if a.only == "native":
        print(json.dumps({"shape": [B, S, Hq, Hk, D], "device": dev_desc, "results": res}))
        return
    A.set_attention_backend("sdpa")
    bench("torch_sdpa", lambda: A.flash_attn_func(q, k, v, causal=True))
    try:
        from flash_attn import flash_attn_func as fa2
        bench("flash_attn2", lambda: fa2(q, k, v, causal=True))
    except Exception as e:
        print("flash_attn unavailable:", e)
    print(json.dumps({"shape": [B, S, Hq, Hk, D], "device": dev_desc, "results": res}))


if __name__ == "__main__":
    main()
