"""Native GPT-2 (the default model of the reference's benchmark, benchmarks/transformer.py:32-68 ``gpt2`` /
``GPT2Block``): learned positions, pre-LN blocks, GELU MLP, tied embeddings.  Linear layers run on the wgmma
GEMM, attention on the flash kernels, the loss on fused linear + cross-entropy; LayerNorm/GELU use PyTorch ops
(Llama-family models are the tuned path)."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import attention as attn_ops
from ..ops.cross_entropy import fused_linear_cross_entropy
from ..ops.linear import linear
from .llama import CausalLMOutput


@dataclass
class GPT2Config:
    vocab_size: int = 50257
    n_positions: int = 1024
    n_embd: int = 768
    n_layer: int = 12
    n_head: int = 12
    layer_norm_epsilon: float = 1e-5
    initializer_range: float = 0.02
    padded_vocab_multiple: int = 128

    @property
    def padded_vocab(self):
        m = self.padded_vocab_multiple
        return (self.vocab_size + m - 1) // m * m


PRESETS = {
    "gpt2": dict(),
    "gpt2-medium": dict(n_embd=1024, n_layer=24, n_head=16),
    "gpt2-large": dict(n_embd=1280, n_layer=36, n_head=20),
    "gpt2-xl": dict(n_embd=1600, n_layer=48, n_head=25),
    "gpt2-tiny": dict(vocab_size=512, n_positions=128, n_embd=128, n_layer=2, n_head=2),
}


class GPT2Block(nn.Module):

    def __init__(self, cfg: GPT2Config, device=None, dtype=None):
        super().__init__()
        kw = dict(device=device, dtype=dtype)
        self.n_head, self.head_dim = cfg.n_head, cfg.n_embd // cfg.n_head
        self.ln_1 = nn.LayerNorm(cfg.n_embd, eps=cfg.layer_norm_epsilon, **kw)
        self.c_attn = nn.Linear(cfg.n_embd, 3 * cfg.n_embd, **kw)
        self.c_proj = nn.Linear(cfg.n_embd, cfg.n_embd, **kw)
        self.ln_2 = nn.LayerNorm(cfg.n_embd, eps=cfg.layer_norm_epsilon, **kw)
        self.c_fc = nn.Linear(cfg.n_embd, 4 * cfg.n_embd, **kw)
        self.c_proj2 = nn.Linear(4 * cfg.n_embd, cfg.n_embd, **kw)

    def forward(self, h, batch, seq_len):
        x = F.layer_norm(h, (h.shape[-1],), self.ln_1.weight, self.ln_1.bias, self.ln_1.eps)
        qkv = linear(x, self.c_attn.weight, self.c_attn.bias)
        a = attn_ops.flash_attn_qkvpacked_tokens(qkv, self.n_head, self.n_head, self.head_dim, batch, seq_len,
                                                 causal=True)
        h = h + linear(a, self.c_proj.weight, self.c_proj.bias)
        x = F.layer_norm(h, (h.shape[-1],), self.ln_2.weight, self.ln_2.bias, self.ln_2.eps)
        m = linear(F.gelu(linear(x, self.c_fc.weight, self.c_fc.bias), approximate="tanh"), self.c_proj2.weight,
                   self.c_proj2.bias)
        return h + m


class GPT2LMHeadModel(nn.Module):

    def __init__(self, cfg: GPT2Config, device=None, dtype=None):
        super().__init__()
        self.config = cfg
        kw = dict(device=device, dtype=dtype)
        self.wte = nn.Embedding(cfg.padded_vocab, cfg.n_embd, **kw)
        self.wpe = nn.Embedding(cfg.n_positions, cfg.n_embd, **kw)
        self.h = nn.ModuleList([GPT2Block(cfg, **kw) for _ in range(cfg.n_layer)])
        self.ln_f = nn.LayerNorm(cfg.n_embd, eps=cfg.layer_norm_epsilon, **kw)
        if device is None or torch.device(device).type != "meta":
            self.reset_parameters()

    @torch.no_grad()
    def reset_parameters(self):
        for n, p in self.named_parameters():
            if p.is_meta:
                continue
            if n.endswith("bias"):
                p.zero_()
            elif "ln_" in n:
                p.fill_(1.0)
            else:
                p.normal_(0.0, self.config.initializer_range)

    @torch.no_grad()
    def load_hf_state_dict(self, sd: dict, strict: bool = True):
        """Load a HuggingFace ``GPT2LMHeadModel`` / ``GPT2Model`` state dict."""
        own = _hf_gpt2_to_native(sd, self.config)
        tgt = self.state_dict()
        own = {k: v.to(tgt[k].dtype) for k, v in own.items()}
        return self.load_state_dict(own, strict=strict)

    def forward(self, input_ids, labels=None, attention_mask=None, return_logits=None, **_unused):
        B, S = input_ids.shape
        pos = torch.arange(S, device=input_ids.device).repeat(B)
        h = self.wte(input_ids.reshape(-1)) + self.wpe(pos)
        for blk in self.h:
            h = blk(h, B, S)
        h = F.layer_norm(h, (h.shape[-1],), self.ln_f.weight, self.ln_f.bias, self.ln_f.eps)
        out = CausalLMOutput()
        if labels is not None:
            lab = torch.full_like(labels, -100)
            lab[:, :-1] = labels[:, 1:]
            out["loss"] = fused_linear_cross_entropy(h, self.wte.weight, lab.reshape(-1),
                                                     valid_vocab=self.config.vocab_size)
        if return_logits or (labels is None and return_logits is None):
            out["logits"] = linear(h, self.wte.weight).view(B, S, -1)[..., :self.config.vocab_size]
        return out


def _hf_gpt2_to_native(sd: dict, cfg: GPT2Config) -> dict:
    """HuggingFace GPT-2 state dict -> ours.  HF stores the projections as Conv1D ([in, out]): transpose them;
    the tied embedding is padded with zero rows up to the aligned vocabulary."""
    out = {}
    g = lambda k: sd[k] if k in sd else sd["transformer." + k]
    wte = g("wte.weight")
    pad = cfg.padded_vocab - wte.shape[0]
    out["wte.weight"] = torch.cat([wte, wte.new_zeros(pad, wte.shape[1])], 0) if pad > 0 else wte
    out["wpe.weight"] = g("wpe.weight")
    out["ln_f.weight"], out["ln_f.bias"] = g("ln_f.weight"), g("ln_f.bias")
    for i in range(cfg.n_layer):
        p, q = f"h.{i}.", f"h.{i}."
        for ln in ("ln_1", "ln_2"):
            out[q + ln + ".weight"], out[q + ln + ".bias"] = g(p + ln + ".weight"), g(p + ln + ".bias")
        for ours, theirs in (("c_attn", "attn.c_attn"), ("c_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"),
                             ("c_proj2", "mlp.c_proj")):
            out[q + ours + ".weight"] = g(p + theirs + ".weight").t().contiguous()
            out[q + ours + ".bias"] = g(p + theirs + ".bias")
    return out


def build_gpt2(name_or_cfg="gpt2", device=None, dtype=None, **overrides) -> GPT2LMHeadModel:
    if isinstance(name_or_cfg, GPT2Config):
        cfg = name_or_cfg
    else:
        kw = dict(PRESETS[name_or_cfg])
        kw.update(overrides)
        cfg = GPT2Config(**kw)
    return GPT2LMHeadModel(cfg, device=device, dtype=dtype)
