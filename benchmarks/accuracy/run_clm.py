#!/usr/bin/env python
"""Causal-LM fine-tuning run used by the accuracy benchmark (counterpart of reference
benchmarks/accuracy/run_clm.py + llama.sh: HF run_clm on Llama-3.2-1B / wikitext, torch-native vs torchacc).

Two arms, selected with ``--impl``:
  native   : torchacc_b200 on its sm_90a kernels (wgmma GEMM, flash attention, fused norm/rope/swiglu/CE/AdamW)
  torch    : the SAME framework code with ``TORCHACC_B200_DISABLE_NATIVE=1`` -> every op runs its plain PyTorch
             reference on the GPU (or CPU)
Both arms share model init, data order and hyper-parameters; the final ``train_loss`` (mean over the last
``--avg_last`` steps) is written to ``--out`` as JSON.  ``run.sh`` asserts |delta| <= 1e-2 like the reference
(benchmarks/accuracy/run.sh:127-132).

Data: a local text file (``--text``; e.g. wikitext-2 train.txt) or, by default, the learnable synthetic Markov corpus
of benchmarks/dataset.py (no network in this sandbox).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--impl", default="native", choices=["native", "torch"])
    p.add_argument("--model", default="llama3.2-1b")
    p.add_argument("--layers", type=int, default=None)
    p.add_argument("--seq_len", type=int, default=1024)
    p.add_argument("--batch_size", type=int, default=4)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--avg_last", type=int, default=20)
    p.add_argument("--lr", type=float, default=3e-4)
    p.add_argument("--fsdp_size", type=int, default=None)
    p.add_argument("--text", default=None)
    p.add_argument("--vocab", type=int, default=4096, help="synthetic corpus vocabulary")
    p.add_argument("--device", default=None)
    p.add_argument("--fp8", action="store_true", help="native arm with Config.compute.fp8 (MX-FP8 linear layers)")
    p.add_argument("--hf", action="store_true",
                   help="train the HuggingFace LlamaForCausalLM of the same geometry through ta.accelerate (what the "
                        "reference's protocol wraps: benchmarks/accuracy/llama.sh) instead of the native model definition")
    p.add_argument("--sp_size", type=int, default=1, help="context-parallel ranks (Ulysses) -- works for --hf too")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if a.impl == "torch":
        os.environ["TORCHACC_B200_DISABLE_NATIVE"] = "1"
        os.environ["TORCHACC_B200_ATTN"] = "reference"
    import torch
    import torchacc_b200 as ta
    from dataset import MarkovLM, TextFileLM, batches
    from torchacc_b200.models import build_llama, llama_config

    rank, world = ta.dist.rank(), ta.dist.world_size()
    device = torch.device(a.device) if a.device else ta.dist.current_device()
    if device.type == "cuda":
        torch.cuda.set_device(device)
    ds = TextFileLM(a.text, a.seq_len) if a.text else MarkovLM(a.vocab, a.seq_len, num_samples=2048, seed=0)
    over = {"vocab_size": 256 if a.text else a.vocab, "max_position_embeddings": max(a.seq_len, 2048)}
    if a.layers:
        over["num_hidden_layers"] = a.layers
    dtype = torch.bfloat16 if device.type == "cuda" else torch.float32
    torch.manual_seed(0)
    lc = llama_config(a.model, **over)
    if a.hf:
        from transformers import LlamaConfig, LlamaForCausalLM
        hc = LlamaConfig(vocab_size=lc.vocab_size, hidden_size=lc.hidden_size, intermediate_size=lc.intermediate_size,
                         num_hidden_layers=lc.num_hidden_layers, num_attention_heads=lc.num_attention_heads,
                         num_key_value_heads=lc.num_key_value_heads, head_dim=lc.head_dim,
                         max_position_embeddings=lc.max_position_embeddings, rope_theta=lc.rope_theta,
                         rms_norm_eps=lc.rms_norm_eps, tie_word_embeddings=False, use_cache=False,
                         attn_implementation="flash_attention_2" if device.type == "cuda" else "eager")
        with torch.device(device):
            model = LlamaForCausalLM(hc).to(dtype)
    else:
        with torch.device(device):
            model = build_llama(lc, dtype=dtype)
    cfg = ta.Config()
    cfg.compute.bf16 = dtype == torch.bfloat16
    cfg.compute.fp8 = bool(a.fp8)
    cfg.memory.gc = True
    cfg.dist.sp.size = a.sp_size
    cfg.dist.fsdp.size = a.fsdp_size or (world // a.sp_size)
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=a.lr, betas=(0.9, 0.95), weight_decay=0.0)
    # ranks of one sp group are replicas: they consume the same batches
    stream = batches(ds, a.batch_size, rank // a.sp_size, world // a.sp_size, seed=1)
    losses = []
    for step in range(a.steps):
        b = {k: v.to(device) for k, v in next(stream).items()}
        out = model(**b)
        loss = out["loss"] if isinstance(out, dict) else out.loss
        loss.backward()
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        losses.append(float(loss.detach()))
        if rank == 0 and (step % 20 == 0 or step == a.steps - 1):
            print(f"[{a.impl}] step {step:4d} loss {losses[-1]:.4f}", flush=True)
    train_loss = sum(losses[-a.avg_last:]) / min(a.avg_last, len(losses))
    res = {"impl": a.impl + ("+fp8" if a.fp8 else "") + ("+hf" if a.hf else ""), "train_loss": train_loss, "first_loss": losses[0], "steps": a.steps,
           "optimal_loss": getattr(ds, "optimal_loss", None)}
    if rank == 0:
        print(json.dumps(res), flush=True)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(res, f)


if __name__ == "__main__":
    main()
