"""Native Llama-family decoder (Llama-2/3, Qwen2-style with QKV bias, Qwen3-style with per-head q / k RMSNorm) built on
the sm_90a op set.

The reference has no model code of its own: it patches HF models (liger kernels, FA) and relies on FlashModels
for TP/CP-aware modules (SURVEY 2.1 #27, #41, 7.1 "native Llama model definition").  This module is that native
definition, laid out for the fused kernels:

* ``qkv_proj``  : one GEMM for q|k|v, RoPE applied in place on its output (with ``qk_norm``: the per-head q / k norm
  and RoPE in one out-of-place kernel), attention reads the packed buffer;
* ``gate_up_proj``: one GEMM for gate|up, SwiGLU kernel on its output;
* RMSNorm fuses the residual add; the loss is fused linear + cross-entropy (no [T, V] logits);
* token-major activations ``[T, H]`` throughout (T = batch * seq), so every op is a plain 2-D GEMM / row kernel.

HF checkpoints load through ``load_hf_state_dict`` (q/k/v and gate/up are concatenated) and export back with
``to_hf_state_dict``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from ..ops import attention as attn_ops
from ..ops.cross_entropy import fused_linear_cross_entropy
from ..ops.linear import linear
from ..ops.rmsnorm import rmsnorm
from ..ops.rope import qk_norm_rope_qkv, rope_qkv_, rope_tables
from ..ops.moe import MoEMLP, load_balancing_loss
from ..ops.swiglu import gate_up_swiglu, swiglu


@dataclass
class LlamaConfig:
    vocab_size: int = 128256
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    head_dim: Optional[int] = None
    rms_norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    rope_scaling: Optional[dict] = None
    max_position_embeddings: int = 8192
    tie_word_embeddings: bool = False
    attention_bias: bool = False          # Qwen2: True (bias on q/k/v)
    sliding_window: Optional[int] = None  # Mistral/Qwen2 style local attention
    initializer_range: float = 0.02
    loss_chunk_tokens: int = 4096
    model_type: str = "llama"
    # mixture of experts (Mixtral style): 0 = dense MLP.  Each token runs num_experts_per_tok experts of width
    # moe_intermediate_size (default: intermediate_size), chosen by a softmax -> top-k router.
    num_experts: int = 0
    num_experts_per_tok: int = 2
    moe_intermediate_size: Optional[int] = None
    norm_topk_prob: bool = True
    router_aux_loss_coef: float = 0.0     # load-balancing loss weight, same scale as HF Mixtral's (0.02 there)
    qk_norm: bool = False                 # Qwen3: RMSNorm of every q and k head (own [head_dim] weights) before RoPE

    def __post_init__(self):
        if self.head_dim is None:
            self.head_dim = self.hidden_size // self.num_attention_heads
        if self.num_experts and self.moe_intermediate_size is None:
            self.moe_intermediate_size = self.intermediate_size

    def _mlp_params(self) -> int:
        """MLP parameters one token uses (for MoE: the router and the k active experts)."""
        h = self.hidden_size
        if self.num_experts:
            return h * self.num_experts + self.num_experts_per_tok * 3 * h * self.moe_intermediate_size
        return 3 * h * self.intermediate_size

    @property
    def qkv_dim(self):
        return (self.num_attention_heads + 2 * self.num_key_value_heads) * self.head_dim

    def num_params(self) -> int:
        """Active parameters per token (all parameters for a dense model)."""
        h, v, L = self.hidden_size, self.vocab_size, self.num_hidden_layers
        per = self.qkv_dim * h + h * self.num_attention_heads * self.head_dim + self._mlp_params() + 2 * h
        if self.attention_bias:
            per += self.qkv_dim
        if self.qk_norm:
            per += 2 * self.head_dim
        return L * per + v * h * (1 if self.tie_word_embeddings else 2) + h

    def flops_per_token(self, seq_len: int, causal: bool = True) -> float:
        """Training FLOPs per token (fwd + bwd = 3x fwd), GEMMs + attention."""
        h, L = self.hidden_size, self.num_hidden_layers
        gemm = 2 * (self.qkv_dim * h + h * self.num_attention_heads * self.head_dim + self._mlp_params()) * L
        gemm += 2 * self.vocab_size * h
        attn = 4 * seq_len * self.num_attention_heads * self.head_dim * L * (0.5 if causal else 1.0)
        return 3.0 * (gemm + attn)


PRESETS = {
    "llama3-8b": dict(),
    "llama3-70b": dict(hidden_size=8192, intermediate_size=28672, num_hidden_layers=80, num_attention_heads=64,
                       num_key_value_heads=8),
    "llama3.2-1b": dict(hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32,
                        num_key_value_heads=8, head_dim=64, tie_word_embeddings=True),
    "llama2-7b": dict(vocab_size=32000, intermediate_size=11008, num_key_value_heads=32, rope_theta=10000.0,
                      max_position_embeddings=4096),
    "qwen2-7b": dict(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                     num_attention_heads=28, num_key_value_heads=4, rope_theta=1000000.0, attention_bias=True,
                     rms_norm_eps=1e-6, model_type="qwen2", max_position_embeddings=32768),
    "mistral-7b": dict(vocab_size=32000, intermediate_size=14336, num_key_value_heads=8, rope_theta=10000.0,
                       sliding_window=4096, max_position_embeddings=32768, model_type="mistral"),
    "qwen2.5-0.5b": dict(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                         num_attention_heads=14, num_key_value_heads=2, head_dim=64, rope_theta=1000000.0,
                         attention_bias=True, rms_norm_eps=1e-6, tie_word_embeddings=True, model_type="qwen2",
                         max_position_embeddings=32768),
    "tiny": dict(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                 num_key_value_heads=2, head_dim=64, max_position_embeddings=512),
    "mixtral-8x7b": dict(vocab_size=32000, intermediate_size=14336, num_key_value_heads=8, rope_theta=1000000.0,
                         max_position_embeddings=32768, num_experts=8, num_experts_per_tok=2, model_type="mixtral"),
    "tiny-moe": dict(vocab_size=512, hidden_size=256, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                     num_key_value_heads=2, head_dim=64, max_position_embeddings=512, num_experts=8,
                     num_experts_per_tok=2, model_type="mixtral"),
}
# Qwen3 / Qwen3-MoE, from the published config.json files
_QWEN3 = dict(vocab_size=151936, head_dim=128, rope_theta=1000000.0, rms_norm_eps=1e-6, max_position_embeddings=40960,
              qk_norm=True, model_type="qwen3")
PRESETS.update({
    "qwen3-0.6b": dict(_QWEN3, hidden_size=1024, intermediate_size=3072, num_hidden_layers=28, num_attention_heads=16,
                       num_key_value_heads=8, tie_word_embeddings=True),
    "qwen3-1.7b": dict(_QWEN3, hidden_size=2048, intermediate_size=6144, num_hidden_layers=28, num_attention_heads=16,
                       num_key_value_heads=8, tie_word_embeddings=True),
    "qwen3-4b": dict(_QWEN3, hidden_size=2560, intermediate_size=9728, num_hidden_layers=36, num_attention_heads=32,
                     num_key_value_heads=8, tie_word_embeddings=True),
    "qwen3-8b": dict(_QWEN3, hidden_size=4096, intermediate_size=12288, num_hidden_layers=36, num_attention_heads=32,
                     num_key_value_heads=8),
    "qwen3-30b-a3b": dict(_QWEN3, hidden_size=2048, intermediate_size=6144, moe_intermediate_size=768,
                          num_hidden_layers=48, num_attention_heads=32, num_key_value_heads=4, num_experts=128,
                          num_experts_per_tok=8, norm_topk_prob=True, router_aux_loss_coef=0.001,
                          model_type="qwen3_moe"),
    "tiny-qwen3": dict(_QWEN3, vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                       num_attention_heads=4, num_key_value_heads=2, head_dim=64, max_position_embeddings=512,
                       tie_word_embeddings=True),
    "tiny-qwen3-moe": dict(_QWEN3, vocab_size=512, hidden_size=256, intermediate_size=512, moe_intermediate_size=128,
                           num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                           max_position_embeddings=512, num_experts=8, num_experts_per_tok=2, norm_topk_prob=True,
                           router_aux_loss_coef=0.001, model_type="qwen3_moe"),
})


def llama_config(name: str, **overrides) -> LlamaConfig:
    kw = dict(PRESETS[name])
    kw.update(overrides)
    return LlamaConfig(**kw)


class ParallelContext:
    """What a layer needs to know about the surrounding parallelism (filled by the TP / CP wrappers)."""

    def __init__(self):
        self.tp = None               # parallel.tp.TPContext when tensor parallel
        self.tp_group = None
        self.tp_size = 1
        self.sequence_parallel = False
        self.cp_mesh = None          # torchacc_b200.parallel mesh for context parallel attention
        self.cp_mode = None          # 'ulysses' | 'ring' | '2d'


class LlamaAttention(nn.Module):

    def __init__(self, cfg: LlamaConfig, layer_idx: int, device=None, dtype=None):
        super().__init__()
        self.cfg = cfg
        self.layer_idx = layer_idx
        self.num_heads = cfg.num_attention_heads
        self.num_kv_heads = cfg.num_key_value_heads
        self.head_dim = cfg.head_dim
        kw = dict(device=device, dtype=dtype)
        self.qkv_proj = nn.Linear(cfg.hidden_size, cfg.qkv_dim, bias=cfg.attention_bias, **kw)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, cfg.hidden_size, bias=False, **kw)
        if cfg.qk_norm:
            self.q_norm = _NormWeight(self.head_dim, cfg.rms_norm_eps, **kw)
            self.k_norm = _NormWeight(self.head_dim, cfg.rms_norm_eps, **kw)

    def forward(self, x, rope, batch, seq_len, position_ids=None, cu_seqlens=None, pctx: Optional[ParallelContext] = None):
        cos, sin = rope
        tp = pctx.tp if pctx is not None else None
        hq, hk = self.num_heads, self.num_kv_heads
        if tp is not None:
            from ..parallel.tp import column_parallel_linear, row_parallel_linear
            qkv = column_parallel_linear(x, self.qkv_proj.weight, self.qkv_proj.bias, tp)   # all-gather -> GEMM
            hq, hk = hq // tp.size, hk // tp.size
        else:
            qkv = linear(x, self.qkv_proj.weight, self.qkv_proj.bias)       # [T, (Hq+2Hk) D]
        window = (-1, -1)
        if self.cfg.sliding_window:
            window = (self.cfg.sliding_window - 1, 0)
        qk_norm = None
        if self.cfg.qk_norm:
            wq, wk = self.q_norm.weight, self.k_norm.weight
            if tp is not None:
                # shared by all heads, so each rank's gradient covers only its own heads: summed over the group
                from ..parallel.tp import tp_head_shared
                wq, wk = tp_head_shared(wq, tp), tp_head_shared(wk, tp)
            qk_norm = (wq, wk, self.q_norm.eps)
        if pctx is not None and pctx.cp_mesh is not None:
            from ..ops.context_parallel import cp_attention_qkvpacked
            o = cp_attention_qkvpacked(qkv, hq, hk, self.head_dim, batch, seq_len, rope, position_ids, pctx,
                                       causal=True, window_size=window, qk_norm=qk_norm)
        else:
            if qk_norm is not None:
                qkv = qk_norm_rope_qkv(qkv, hq, hk, self.head_dim, *qk_norm, cos, sin, position_ids, seq_len)
            else:
                qkv = rope_qkv_(qkv, hq, hk, self.head_dim, cos, sin, position_ids, seq_len)
            o = attn_ops.flash_attn_qkvpacked_tokens(qkv, hq, hk, self.head_dim, batch, seq_len, causal=True,
                                                     window_size=window, cu_seqlens=cu_seqlens)
        if tp is not None:
            return row_parallel_linear(o, self.o_proj.weight, tp)           # GEMM -> reduce-scatter
        return linear(o, self.o_proj.weight, None)


class LlamaMLP(nn.Module):

    def __init__(self, cfg: LlamaConfig, device=None, dtype=None):
        super().__init__()
        kw = dict(device=device, dtype=dtype)
        self.gate_up_proj = nn.Linear(cfg.hidden_size, 2 * cfg.intermediate_size, bias=False, **kw)
        self.down_proj = nn.Linear(cfg.intermediate_size, cfg.hidden_size, bias=False, **kw)

    def forward(self, x, pctx=None, residual=None):
        """``residual`` (the skip branch) is added in the down-projection's GEMM epilogue."""
        tp = pctx.tp if pctx is not None else None
        if tp is not None:
            from ..parallel.tp import column_parallel_linear, row_parallel_linear
            m = row_parallel_linear(swiglu(column_parallel_linear(x, self.gate_up_proj.weight, None, tp)),
                                    self.down_proj.weight, tp)
            return m if residual is None else residual + m
        # gate|up GEMM with the SwiGLU activation in its epilogue (no [T, 2F] round trip), down projection with the
        # residual add in its epilogue
        return linear(gate_up_swiglu(x, self.gate_up_proj.weight), self.down_proj.weight, residual=residual)


class LlamaDecoderLayer(nn.Module):
    """h -> h + attn(norm(h)) -> (+ mlp(norm(.))).  Single tensor in / out so FSDP units, gradient checkpointing
    and pipeline stages can wrap it uniformly."""

    def __init__(self, cfg: LlamaConfig, layer_idx: int, device=None, dtype=None):
        super().__init__()
        kw = dict(device=device, dtype=dtype)
        self.input_layernorm = _NormWeight(cfg.hidden_size, cfg.rms_norm_eps, **kw)
        self.self_attn = LlamaAttention(cfg, layer_idx, **kw)
        self.post_attention_layernorm = _NormWeight(cfg.hidden_size, cfg.rms_norm_eps, **kw)
        if cfg.num_experts:
            self.mlp = MoEMLP(cfg.hidden_size, cfg.moe_intermediate_size, cfg.num_experts, cfg.num_experts_per_tok,
                              cfg.norm_topk_prob, **kw)
        else:
            self.mlp = LlamaMLP(cfg, **kw)

    def forward(self, h, rope, batch, seq_len, position_ids=None, cu_seqlens=None, pctx=None):
        w1, w2 = self.input_layernorm.weight, self.post_attention_layernorm.weight
        if pctx is not None and pctx.tp is not None:
            from ..parallel.tp import tp_replicated
            w1, w2 = tp_replicated(w1, pctx.tp), tp_replicated(w2, pctx.tp)
        # no stand-alone elementwise adds: the skip branch leaves norm 1 as a pass-through output (its gradient is
        # summed inside the norm's backward kernel), the attention residual is fused into norm 2, the MLP residual
        # into the down-projection's GEMM epilogue
        y, h_skip = rmsnorm(h, w1, self.input_layernorm.eps, passthrough=True)
        a = self.self_attn(y, rope, batch, seq_len, position_ids, cu_seqlens, pctx)
        y2, h2 = rmsnorm(a, w2, self.post_attention_layernorm.eps, residual=h_skip)
        if isinstance(self.mlp, MoEMLP):
            return self.mlp(y2, residual=h2)          # residual added in the combine kernel
        return self.mlp(y2, pctx, residual=h2)


class _NormWeight(nn.Module):
    """RMSNorm parameter holder (the math lives in ops.rmsnorm so the residual add can be fused by the caller)."""

    def __init__(self, hidden, eps, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden, device=device, dtype=dtype))
        self.eps = eps

    def forward(self, x, residual=None):
        y, h = rmsnorm(x, self.weight, self.eps, residual)
        return y if residual is None else (y, h)


class LlamaModel(nn.Module):

    def __init__(self, cfg: LlamaConfig, device=None, dtype=None):
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=dtype)
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size, **kw)
        self.layers = nn.ModuleList([LlamaDecoderLayer(cfg, i, **kw) for i in range(cfg.num_hidden_layers)])
        self.norm = _NormWeight(cfg.hidden_size, cfg.rms_norm_eps, **kw)
        self._rope = None
        self.pctx = ParallelContext()
        self.gradient_checkpointing = False

    def rope(self, device):
        if self._rope is None or self._rope[0].device != device:
            self._rope = rope_tables(self.cfg.max_position_embeddings, self.cfg.head_dim, self.cfg.rope_theta, device,
                                     self.cfg.rope_scaling)
        return self._rope

    def forward(self, input_ids, position_ids=None, cu_seqlens=None):
        if self.pctx.cp_mesh is not None:
            # context parallel: every rank receives the full sequence and keeps its own shard of the tokens
            from ..ops.context_parallel import cp_shard_sequence
            input_ids = cp_shard_sequence(input_ids, 1, self.pctx)
            if position_ids is not None:
                position_ids = cp_shard_sequence(position_ids, 1, self.pctx)
        B, S = input_ids.shape
        h = self.embed_tokens(input_ids.reshape(-1))                          # [T, H]
        rope = self.rope(h.device)
        s_full = S * (self.pctx.cp_mesh.get_sp_num() if self.pctx.cp_mesh is not None else 1)
        if s_full > rope[0].shape[0]:
            raise ValueError(f"sequence length {s_full} exceeds max_position_embeddings {rope[0].shape[0]}")
        pos = position_ids.reshape(-1).to(torch.int32) if position_ids is not None else None
        tp = self.pctx.tp
        wn = self.norm.weight
        if tp is not None and tp.sequence_parallel:
            from ..parallel.tp import scatter_tokens, tp_replicated
            h = scatter_tokens(h, tp)                       # residual stream is token-sharded between the linears
            wn = tp_replicated(wn, tp)
        for layer in self.layers:
            h = layer(h, rope, B, S, pos, cu_seqlens, self.pctx)
        y, _ = rmsnorm(h, wn, self.norm.eps)
        return y


class CausalLMOutput(dict):
    """Dict with attribute access (``out.loss`` / ``out['loss']``), like HF model outputs."""
    __getattr__ = dict.get


class LlamaForCausalLM(nn.Module):

    def __init__(self, cfg: LlamaConfig, device=None, dtype=None):
        super().__init__()
        self.config = cfg
        self.model = LlamaModel(cfg, device=device, dtype=dtype)
        self.lm_head = nn.Linear(cfg.hidden_size, cfg.vocab_size, bias=False, device=device, dtype=dtype)
        if cfg.tie_word_embeddings:
            self.lm_head.weight = self.model.embed_tokens.weight
        if device is None or torch.device(device).type != "meta":
            self.reset_parameters()

    @torch.no_grad()
    def reset_parameters(self):
        std = self.config.initializer_range
        for name, p in self.named_parameters():
            if p.is_meta:
                continue
            if name.endswith("layernorm.weight") or name.endswith("norm.weight"):
                p.fill_(1.0)
            elif name.endswith(".bias"):
                p.zero_()
            else:
                p.normal_(0.0, std)

    def forward(self, input_ids, labels=None, position_ids=None, attention_mask=None, cu_seqlens=None,
                return_logits: Optional[bool] = None, shift_labels: bool = True, n_valid_total=None, **_unused):
        """``labels`` follow the HF convention (same shape as input_ids, shifted internally, -100 ignored).
        With labels the loss is computed by fused linear+CE and logits are not materialised unless
        ``return_logits=True``."""
        B, S = input_ids.shape
        if attention_mask is not None and position_ids is None and cu_seqlens is None \
                and not bool(attention_mask.all()):
            # right-padded batch: padded keys are never visible under causal masking to valid queries of the same
            # row; padded query rows are ignored by the loss (labels = -100 expected).
            pass
        hidden = self.model(input_ids, position_ids, cu_seqlens)              # [T, H]
        out = CausalLMOutput()
        if labels is not None:
            if shift_labels:
                lab = torch.full_like(labels, -100)
                lab[:, :-1] = labels[:, 1:]
                if position_ids is not None:  # packed sequences: do not predict across a sequence boundary
                    nxt_is_start = torch.zeros_like(labels, dtype=torch.bool)
                    nxt_is_start[:, :-1] = position_ids[:, 1:] == 0
                    lab = lab.masked_fill(nxt_is_start, -100)
            else:
                lab = labels
            if self.model.pctx.cp_mesh is not None:
                from ..ops.context_parallel import cp_shard_sequence
                if n_valid_total is None:
                    # every rank holds the full labels: normalise by (global valid tokens / sp) so that the mean of
                    # the per-rank losses (and of their gradients over the replica group) is the exact global loss
                    n_valid_total = (lab != -100).sum().clamp(min=1).float() / self.model.pctx.cp_mesh.get_sp_num()
                lab = cp_shard_sequence(lab, 1, self.model.pctx)
            tp = self.model.pctx.tp
            if tp is not None:
                from ..parallel.tp import gather_tokens, vocab_parallel_cross_entropy
                hid = gather_tokens(hidden, tp) if tp.sequence_parallel else hidden
                out["loss"] = vocab_parallel_cross_entropy(hid, self.lm_head.weight, lab.reshape(-1), tp,
                                                          n_valid_total=n_valid_total)
            else:
                out["loss"] = fused_linear_cross_entropy(hidden, self.lm_head.weight, lab.reshape(-1),
                                                         chunk_tokens=self.config.loss_chunk_tokens,
                                                         n_valid_total=n_valid_total)
            if self.config.num_experts and self.config.router_aux_loss_coef:
                out["aux_loss"] = self.router_aux_loss()
                out["loss"] = out["loss"] + self.config.router_aux_loss_coef * out["aux_loss"]
        if return_logits or (labels is None and return_logits is None):
            tp = self.model.pctx.tp
            if self.model.pctx.cp_mesh is not None:
                S = S // self.model.pctx.cp_mesh.get_sp_num()      # logits of the local sequence shard
            if tp is not None:
                from ..parallel.tp import gather_tokens
                hid = gather_tokens(hidden, tp) if tp.sequence_parallel else hidden
                local = linear(hid, self.lm_head.weight)                      # [T, V/tp]
                parts = [torch.empty_like(local) for _ in range(tp.size)]
                torch.distributed.all_gather(parts, local.contiguous(), group=tp.group)
                out["logits"] = torch.cat(parts, -1).view(B, S, -1)
            else:
                out["logits"] = linear(hidden, self.lm_head.weight).view(B, S, -1)
        return out

    def router_aux_loss(self) -> torch.Tensor:
        """Load-balancing loss of the latest forward over all MoE layers (HF Mixtral's definition and scale)."""
        layers = [l.mlp for l in self.model.layers if isinstance(l.mlp, MoEMLP)]
        return load_balancing_loss([m.last_router_logits for m in layers], [m.last_counts for m in layers],
                                   self.config.num_experts)

    # ---- HF interop -------------------------------------------------------------------------------------
    @torch.no_grad()
    def load_hf_state_dict(self, sd: dict, strict: bool = True):
        """Load a HuggingFace Llama/Qwen2/Qwen3 state dict (separate q/k/v and gate/up projections), or a Mixtral /
        Qwen3-MoE one (``mlp.gate.weight``, ``mlp.experts.gate_up_proj``, ``mlp.experts.down_proj``: the same names
        here)."""
        own = {}
        L = self.config.num_hidden_layers
        g = lambda k: sd[k]
        own["model.embed_tokens.weight"] = g("model.embed_tokens.weight")
        own["model.norm.weight"] = g("model.norm.weight")
        # tied: lm_head.weight is the embedding parameter, listed under both names by state_dict()
        own["lm_head.weight"] = sd.get("lm_head.weight", sd["model.embed_tokens.weight"])
        for i in range(L):
            p = f"model.layers.{i}."
            own[p + "input_layernorm.weight"] = g(p + "input_layernorm.weight")
            own[p + "post_attention_layernorm.weight"] = g(p + "post_attention_layernorm.weight")
            own[p + "self_attn.qkv_proj.weight"] = torch.cat(
                [g(p + "self_attn.q_proj.weight"), g(p + "self_attn.k_proj.weight"), g(p + "self_attn.v_proj.weight")], 0)
            if self.config.attention_bias:
                own[p + "self_attn.qkv_proj.bias"] = torch.cat(
                    [g(p + "self_attn.q_proj.bias"), g(p + "self_attn.k_proj.bias"), g(p + "self_attn.v_proj.bias")], 0)
            own[p + "self_attn.o_proj.weight"] = g(p + "self_attn.o_proj.weight")
            if self.config.qk_norm:
                own[p + "self_attn.q_norm.weight"] = g(p + "self_attn.q_norm.weight")
                own[p + "self_attn.k_norm.weight"] = g(p + "self_attn.k_norm.weight")
            if self.config.num_experts:
                for name in ("mlp.gate.weight", "mlp.experts.gate_up_proj", "mlp.experts.down_proj"):
                    own[p + name] = g(p + name)
                continue
            own[p + "mlp.gate_up_proj.weight"] = torch.cat([g(p + "mlp.gate_proj.weight"), g(p + "mlp.up_proj.weight")], 0)
            own[p + "mlp.down_proj.weight"] = g(p + "mlp.down_proj.weight")
        return self.load_state_dict(own, strict=strict)

    @torch.no_grad()
    def to_hf_state_dict(self) -> dict:
        cfg = self.config
        sd = self.state_dict()
        out = {}
        qd, kd = cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
        for k, v in sd.items():
            if k.endswith("self_attn.qkv_proj.weight") or k.endswith("self_attn.qkv_proj.bias"):
                base, kind = k.rsplit("qkv_proj.", 1)
                q, kk, vv = v.split([qd, kd, kd], 0)
                out[base + "q_proj." + kind], out[base + "k_proj." + kind], out[base + "v_proj." + kind] = q, kk, vv
            elif k.endswith("mlp.gate_up_proj.weight"):
                base = k[:-len("gate_up_proj.weight")]
                gte, up = v.chunk(2, 0)
                out[base + "gate_proj.weight"], out[base + "up_proj.weight"] = gte, up
            else:
                out[k] = v
        return out


def build_llama(name_or_cfg, device=None, dtype=None, **overrides) -> LlamaForCausalLM:
    cfg = name_or_cfg if isinstance(name_or_cfg, LlamaConfig) else llama_config(name_or_cfg, **overrides)
    return LlamaForCausalLM(cfg, device=device, dtype=dtype)


class LlamaPipelineStage(nn.Module):
    """One pipeline stage of a Llama model: optional embedding, a contiguous range of decoder layers, optional
    final norm + lm_head/loss.  Stage boundaries carry ``hidden`` as [B, S, H]."""

    def __init__(self, lm: LlamaForCausalLM, start: int, end: int, first: bool, last: bool):
        super().__init__()
        self.config = lm.config
        self.first, self.last = first, last
        self.layers = nn.ModuleList(list(lm.model.layers[start:end]))
        self.layer_offset = start
        if first:
            self.embed_tokens = lm.model.embed_tokens
        if last:
            self.norm = lm.model.norm
            self.lm_head = lm.lm_head
        self._owner = [lm.model]     # rope tables / parallel context live on the original LlamaModel

    def forward(self, input_ids=None, hidden=None, labels=None, position_ids=None, cu_seqlens=None,
                return_logits=None, **_unused):
        core = self._owner[0]
        pctx = core.pctx
        if pctx.cp_mesh is not None:
            raise NotImplementedError("pipeline x context parallelism: shard the sequence outside the pipeline")
        if self.first:
            B, S = input_ids.shape
            h = self.embed_tokens(input_ids.reshape(-1))
        else:
            B, S = hidden.shape[0], hidden.shape[1]
            h = hidden.reshape(B * S, hidden.shape[-1])
        rope = core.rope(h.device)
        pos = position_ids.reshape(-1).to(torch.int32) if position_ids is not None else None
        # tensor parallelism inside a stage: the boundary tensor is the full (tp-replicated) hidden state; with
        # sequence parallelism the residual stream is token-sharded between scatter (stage entry) and gather (exit)
        tp = pctx.tp
        sp = tp is not None and tp.sequence_parallel
        if sp:
            from ..parallel.tp import gather_tokens, scatter_tokens, tp_replicated
            h = scatter_tokens(h, tp)
        for layer in self.layers:
            h = layer(h, rope, B, S, pos, cu_seqlens, pctx)
        if not self.last:
            if sp:
                from ..parallel.tp import gather_tokens_replicated_grad
                h = gather_tokens_replicated_grad(h, tp)
            return {"hidden": h.view(B, S, -1)}
        wn = tp_replicated(self.norm.weight, tp) if sp else self.norm.weight
        y, _ = rmsnorm(h, wn, self.norm.eps)
        out = CausalLMOutput()
        if labels is not None:
            lab = torch.full_like(labels, -100)
            lab[:, :-1] = labels[:, 1:]
            if tp is not None:      # lm_head is vocab-sharded: labels outside the local slice must never index it
                from ..parallel.tp import gather_tokens, vocab_parallel_cross_entropy
                hid = gather_tokens(y, tp) if sp else y
                out["loss"] = vocab_parallel_cross_entropy(hid, self.lm_head.weight, lab.reshape(-1), tp)
            else:
                out["loss"] = fused_linear_cross_entropy(y, self.lm_head.weight, lab.reshape(-1),
                                                         chunk_tokens=self.config.loss_chunk_tokens)
        if return_logits or (labels is None and return_logits is None):
            if tp is not None:
                from ..parallel.tp import gather_tokens
                hid = gather_tokens(y, tp) if sp else y
                local = linear(hid, self.lm_head.weight)
                parts = [torch.empty_like(local) for _ in range(tp.size)]
                torch.distributed.all_gather(parts, local.contiguous(), group=tp.group)
                out["logits"] = torch.cat(parts, -1).view(B, S, -1)
            else:
                out["logits"] = linear(y, self.lm_head.weight).view(B, S, -1)
        return out


def _llama_pipeline_stages(self: LlamaForCausalLM, split_names):
    """Native pipeline protocol (see parallel/pp/partition.py): split points must name decoder layers
    (``model.layers.K``), ``model.norm`` or ``lm_head``."""
    from ..parallel.pp.partition import StageSpec
    L = self.config.num_hidden_layers
    cuts = []
    for n in split_names:
        if n.startswith("model.layers."):
            cuts.append(int(n.split(".")[2]))
        elif n in ("model.norm", "lm_head"):
            cuts.append(L)
        else:
            raise ValueError(f"unsupported Llama split point '{n}' (use model.layers.K, model.norm or lm_head)")
    if cuts != sorted(cuts):
        raise ValueError("split points must be listed in execution order")
    bounds = [0] + cuts + [L]
    n = len(bounds) - 1
    if n > 1 and self.config.tie_word_embeddings:
        # the first-stage embedding and the last-stage lm_head would become independent copies whose gradients are
        # never combined (the reference's ReduceTiedGrads is dead code too, executor.py:140-144): refuse loudly
        raise ValueError("pipeline parallelism with tie_word_embeddings=True is not supported: the tied weight would "
                         "live on two stages without gradient synchronisation; untie it (copy into lm_head) first")
    specs = []
    for i in range(n):
        st = LlamaPipelineStage(self, bounds[i], bounds[i + 1], i == 0, i == n - 1)
        specs.append(StageSpec(index=i, module=st,
                               recv_names=[] if i == 0 else ["hidden"],
                               load_names=(["input_ids"] if i == 0 else []) + (["labels"] if i == n - 1 else []) +
                               ["position_ids"],
                               send_names=[] if i == n - 1 else ["hidden"]))
    return specs


LlamaForCausalLM.pipeline_stages = _llama_pipeline_stages
