"""One MoE layer's experts, forward + backward, on the native grouped GEMMs vs HF's ``grouped_mm`` experts forward.

Shapes: Mixtral-8x7B (T=8192, H=4096, F=14336, E=8, k=2) and Qwen3-30B-A3B (T=8192, H=2048, F=768, E=128, k=8), with
seeded routing.  Times come from CUDA events (best and median of --iters after --warmup); the two paths alternate in
the same run.  TFLOP/s count the real (token, expert) pairs, not the padded rows.  Prints one JSON line per shape.

    python benchmarks/moe_bench.py [--iters 20] [--warmup 5] [--shapes mixtral,qwen3] [--fp8]

``--fp8`` adds the MX-FP8 experts (``compute.fp8``), timed alternating with the bf16 native experts, with the peak
memory of one forward + backward of each and the fp8 output's relative difference from the bf16 one.  The fp8 times
include the quantisation passes, over the padded capacity rows too.

``--model-step PRESET`` instead times training steps (forward + backward, no optimizer) of the preset cut to
``--layers`` decoder layers, through ``accelerate`` with FSDP and activation checkpointing of every decoder layer, with
bf16 experts and then with fp8 experts, and reports the peak memory of a step above what the model holds before it.

    python benchmarks/moe_bench.py --model-step qwen3-30b-a3b --layers 4 [--tokens 8192]
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


def peak_mib(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def run(shape, iters, warmup, with_fp8=False):
    from torchacc_b200.ops import fp8
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

    def in_fp8(fn):
        def run_fp8():
            fp8.enable(True)
            try:
                return fn()
            finally:
                fp8.enable(False)
        return run_fp8

    fp8.enable(False)
    diff = (ours_fwd().float() - hf_fwd().float()).abs().max().item()
    t_ours_f, t_hf_f, t_ours_fb, t_fp8_f, t_fp8_fb = [], [], [], [], []
    for _ in range(2):   # alternate the paths
        t_ours_f += time_it(ours_fwd, iters // 2, warmup)
        t_hf_f += time_it(hf_fwd, iters // 2, warmup)
        t_ours_fb += time_it(ours_fwd_bwd, iters // 2, warmup)
        if with_fp8:
            t_fp8_f += time_it(in_fp8(ours_fwd), iters // 2, warmup)
            t_fp8_fb += time_it(in_fp8(ours_fwd_bwd), iters // 2, warmup)
    idx = MoEIndex(ids, E)
    real_rows = T * k
    padded_rows = int(idx.offsets[-1].item())
    name, limit = card()

    def stats(ts, backward):
        best, med = min(ts), statistics.median(ts)
        return dict(best_ms=round(best, 3), median_ms=round(med, 3),
                    tflops_best=round(flops(T, H, Fd, k, backward) / best / 1e9, 1),
                    tflops_median=round(flops(T, H, Fd, k, backward) / med / 1e9, 1))

    res = dict(shape=shape, T=T, H=H, F=Fd, E=E, k=k, gpu=name, power_limit=limit,
               native_fwd=stats(t_ours_f, False), hf_grouped_mm_fwd=stats(t_hf_f, False),
               native_fwd_bwd=stats(t_ours_fb, True), padding_overhead=round(padded_rows / real_rows - 1, 4),
               max_abs_diff_vs_hf=diff, iters=len(t_ours_f))
    if with_fp8:
        from torchacc_b200.ops import moe as moe_mod
        calls = moe_mod.FP8_EXPERT_CALLS
        ref = ours_fwd().float()
        got = in_fp8(ours_fwd)().float()
        assert moe_mod.FP8_EXPERT_CALLS == calls + 1, "the fp8 experts did not run"
        res.update(fp8_fwd=stats(t_fp8_f, False), fp8_fwd_bwd=stats(t_fp8_fb, True),
                   fp8_vs_bf16_fwd=round(statistics.median(t_fp8_f) / statistics.median(t_ours_f) - 1, 4),
                   fp8_vs_bf16_fwd_bwd=round(statistics.median(t_fp8_fb) / statistics.median(t_ours_fb) - 1, 4),
                   fp8_rel_diff_vs_bf16=round(float((got - ref).norm() / ref.norm()), 5),
                   peak_mib_bf16_fwd_bwd=peak_mib(ours_fwd_bwd), peak_mib_fp8_fwd_bwd=peak_mib(in_fp8(ours_fwd_bwd)))
    return res


def model_step(preset, layers, tokens, iters, warmup):
    import gc
    import torchacc_b200 as ta
    from torchacc_b200.models import build_llama
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops import moe as moe_mod
    dev = torch.device("cuda", 0)
    res = dict(model=preset, layers=layers, tokens=tokens, parallelism="fsdp1+gc")
    for name, use_fp8 in (("bf16", False), ("fp8", True)):   # one model at a time: two would not both fit
        torch.manual_seed(0)
        with torch.device(dev):
            model = build_llama(preset, dtype=torch.bfloat16, num_hidden_layers=layers)
        vocab = model.config.vocab_size
        cfg = ta.Config()
        cfg.compute.bf16 = True
        cfg.compute.fp8 = use_fp8
        cfg.memory.gc = True
        cfg.memory.gc_cls = {"LlamaDecoderLayer"}
        cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
        model = ta.accelerate(model, config=cfg)
        g = torch.Generator(device=dev).manual_seed(0)
        ids = torch.randint(0, vocab, (max(tokens // 4096, 1), min(tokens, 4096)), device=dev, generator=g)

        def step():
            out = model(input_ids=ids, labels=ids)
            out["loss"].backward()
            model.zero_grad()

        calls = moe_mod.FP8_EXPERT_CALLS
        ms = time_it(step, iters, warmup)
        assert (moe_mod.FP8_EXPERT_CALLS > calls) == use_fp8, "the experts did not take the expected path"
        res[name] = dict(median_ms=round(statistics.median(ms), 2), best_ms=round(min(ms), 2),
                         peak_step_mib=peak_mib(step))
        fp8.enable(False)
        del model, step
        gc.collect()
        torch.cuda.empty_cache()
    res["gpu"], res["power_limit"] = card()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="mixtral,qwen3")
    ap.add_argument("--fp8", action="store_true", help="also time the MX-FP8 experts against the bf16 ones")
    ap.add_argument("--model-step", default=None, metavar="PRESET", help="time training steps of a MoE preset instead")
    ap.add_argument("--layers", type=int, default=4, help="decoder layers of --model-step")
    ap.add_argument("--tokens", type=int, default=8192, help="tokens per step of --model-step (sequences of 4096)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_bench.py needs a GPU")
    if a.model_step:
        print(json.dumps(model_step(a.model_step, a.layers, a.tokens, a.iters, a.warmup)), flush=True)
        return
    for s in a.shapes.split(","):
        print(json.dumps(run(s, a.iters, a.warmup, a.fp8)), flush=True)


if __name__ == "__main__":
    main()
