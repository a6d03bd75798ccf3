"""One MoE layer's experts, forward + backward, on the native grouped GEMMs vs HF's ``grouped_mm`` experts forward.

Shapes: Mixtral-8x7B (T=8192, H=4096, F=14336, E=8, k=2) and Qwen3-30B-A3B (T=8192, H=2048, F=768, E=128, k=8), with
seeded routing.  Times come from CUDA events (best and median of --iters after --warmup); the two paths alternate in
the same run.  TFLOP/s count the real (token, expert) pairs, not the padded rows.  Prints one JSON line per shape.

    python benchmarks/moe_bench.py [--iters 20] [--warmup 5] [--shapes mixtral,qwen3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"mixtral": dict(T=8192, H=4096, F=14336, E=8, k=2),
          "qwen3": dict(T=8192, H=2048, F=768, E=128, k=8)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        limit = "unknown"
    return name, limit


def flops(T, H, F, k, backward):
    pairs = T * k
    fwd = 2 * pairs * H * (2 * F) + 2 * pairs * F * H
    return fwd * (3 if backward else 1)


def time_it(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def run(shape, iters, warmup):
    from torchacc_b200.ops.moe import MoEIndex, moe_experts
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts
    s = SHAPES[shape]
    T, H, Fd, E, k = s["T"], s["H"], s["F"], s["E"], s["k"]
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(T, H, device=dev, dtype=torch.bfloat16, generator=g)
    logits = torch.randn(T, E, device=dev, generator=g)
    w, ids = torch.topk(torch.softmax(logits, -1), k, -1)
    w = w / w.sum(-1, keepdim=True)
    cfg = MixtralConfig(hidden_size=H, intermediate_size=Fd, num_local_experts=E, num_experts_per_tok=k)
    cfg._experts_implementation = "grouped_mm"
    hf = MixtralExperts(cfg).to(dev, torch.bfloat16)
    with torch.no_grad():
        hf.gate_up_proj.normal_(0, H ** -0.5, generator=g)
        hf.down_proj.normal_(0, Fd ** -0.5, generator=g)
    wgu = hf.gate_up_proj.detach().requires_grad_(True)
    wd = hf.down_proj.detach().requires_grad_(True)
    xg = x.clone().requires_grad_(True)
    dout = torch.randn(T, H, device=dev, dtype=torch.bfloat16, generator=g)

    def ours_fwd():
        with torch.no_grad():
            return moe_experts(x, ids, w, wgu, wd)

    def ours_fwd_bwd():
        out = moe_experts(xg, ids, w, wgu, wd)
        out.backward(dout)

    def hf_fwd():
        with torch.no_grad():
            return hf(x, ids, w.to(torch.bfloat16))

    diff = (ours_fwd().float() - hf_fwd().float()).abs().max().item()
    t_ours_f, t_hf_f, t_ours_fb = [], [], []
    for _ in range(2):   # alternate the paths
        t_ours_f += time_it(ours_fwd, iters // 2, warmup)
        t_hf_f += time_it(hf_fwd, iters // 2, warmup)
        t_ours_fb += time_it(ours_fwd_bwd, iters // 2, warmup)
    idx = MoEIndex(ids, E)
    real_rows = T * k
    padded_rows = int(idx.offsets[-1].item())
    name, limit = card()

    def stats(ts, backward):
        best, med = min(ts), statistics.median(ts)
        return dict(best_ms=round(best, 3), median_ms=round(med, 3),
                    tflops_best=round(flops(T, H, Fd, k, backward) / best / 1e9, 1))

    return dict(shape=shape, T=T, H=H, F=Fd, E=E, k=k, gpu=name, power_limit=limit,
                native_fwd=stats(t_ours_f, False), hf_grouped_mm_fwd=stats(t_hf_f, False),
                native_fwd_bwd=stats(t_ours_fb, True), padding_overhead=round(padded_rows / real_rows - 1, 4),
                max_abs_diff_vs_hf=diff, iters=len(t_ours_f))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="mixtral,qwen3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_bench.py needs a GPU")
    for s in a.shapes.split(","):
        print(json.dumps(run(s, a.iters, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
