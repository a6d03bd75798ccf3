"""Qwen3 / Qwen3-MoE on CPU: the per-head q / k RMSNorm + RoPE op's reference path, the native presets, HF checkpoint
interop, the HF Qwen3 kernel patches and the parallel engines (gloo) against one process."""
import pytest
import torch

from dist_utils import run_distributed


# ---------------------------------------------------------------------------------------------------------------------
# op
# ---------------------------------------------------------------------------------------------------------------------
def test_qk_norm_rope_reference_math():
    """Off the GPU the op is rmsnorm_ref per head then _rope_ref: checked against the contract written out."""
    from torchacc_b200.ops import qk_norm_rope_qkv, rope_tables
    g = torch.Generator().manual_seed(0)
    T, hq, hk, D, eps = 10, 3, 1, 16, 1e-6
    cos, sin = rope_tables(64, D, 1e6)
    cos, sin = cos.double(), sin.double()
    qkv = torch.randn(T, (hq + 2 * hk) * D, generator=g, dtype=torch.float64)
    wq = 1 + 0.1 * torch.randn(D, generator=g, dtype=torch.float64)
    wk = 1 + 0.1 * torch.randn(D, generator=g, dtype=torch.float64)
    pos = torch.randint(0, 64, (T,), generator=g)
    out = qk_norm_rope_qkv(qkv, hq, hk, D, wq, wk, eps, cos, sin, pos, 64)
    x = qkv.view(T, hq + 2 * hk, D)
    z = x * torch.rsqrt(x.square().mean(-1, keepdim=True) + eps)
    z = torch.cat([z[:, :hq] * wq, z[:, hq:hq + hk] * wk], 1)
    c, s = cos[pos.long()].unsqueeze(1), sin[pos.long()].unsqueeze(1)
    z1, z2 = z[..., :D // 2], z[..., D // 2:]
    ref = torch.cat([torch.cat([z1 * c - z2 * s, z2 * c + z1 * s], -1), x[:, hq + hk:]], 1).reshape(T, -1)
    assert torch.allclose(out, ref, atol=1e-12)
    # sequential positions: t % seq_len
    out_seq = qk_norm_rope_qkv(qkv, hq, hk, D, wq, wk, eps, cos, sin, None, 5)
    ref_seq = qk_norm_rope_qkv(qkv, hq, hk, D, wq, wk, eps, cos, sin, torch.arange(T) % 5, 5)
    assert torch.equal(out_seq, ref_seq)
    # autograd through the composition gives the backward the kernel implements: u = rope^-1(g), xhat = x rstd,
    # dx = rstd (u w - xhat mean(u w xhat)), dw = sum u xhat (the composition runs in fp32: fp32 tolerances)
    a, b, cc = (t.clone().requires_grad_() for t in (qkv, wq, wk))
    gout = torch.randn(out.shape, generator=g, dtype=torch.float64)
    qk_norm_rope_qkv(a, hq, hk, D, b, cc, eps, cos, sin, pos, 64).backward(gout)
    g3 = gout.view(T, hq + 2 * hk, D)
    g1, g2 = g3[..., :D // 2], g3[..., D // 2:]
    u = torch.cat([g1 * c + g2 * s, g2 * c - g1 * s], -1)[:, :hq + hk]
    rstd = torch.rsqrt(x[:, :hq + hk].square().mean(-1, keepdim=True) + eps)
    xh = x[:, :hq + hk] * rstd
    w = torch.cat([wq.expand(hq, D), wk.expand(hk, D)], 0)
    dx = rstd * (u * w - xh * (u * w * xh).mean(-1, keepdim=True))
    assert torch.allclose(a.grad.view(T, -1, D)[:, :hq + hk], dx, atol=1e-5)
    assert torch.equal(a.grad.view(T, -1, D)[:, hq + hk:], g3[:, hq + hk:])
    assert torch.allclose(b.grad, (u * xh)[:, :hq].sum((0, 1)), atol=1e-5)
    assert torch.allclose(cc.grad, (u * xh)[:, hq:].sum((0, 1)), atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# presets
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,published", [("qwen3-0.6b", 0.6e9), ("qwen3-1.7b", 1.7e9), ("qwen3-4b", 4.0e9),
                                            ("qwen3-8b", 8.2e9), ("qwen3-30b-a3b", 3.3e9)])
def test_qwen3_preset_parameter_counts(name, published):
    """Parameters (activated parameters for 30B-A3B) within 2 % of the published totals."""
    from torchacc_b200.models import llama_config
    cfg = llama_config(name)
    assert cfg.qk_norm and cfg.head_dim == 128 and cfg.vocab_size == 151936 and not cfg.attention_bias
    assert abs(cfg.num_params() / published - 1) < 0.02, cfg.num_params()


def test_qk_norm_weights_are_counted_and_named():
    from torchacc_b200.models import build_llama, llama_config
    m = build_llama("tiny-qwen3")
    names = {n: p.shape for n, p in m.named_parameters()}
    assert names["model.layers.1.self_attn.q_norm.weight"] == (64,)
    assert names["model.layers.1.self_attn.k_norm.weight"] == (64,)
    cfg = llama_config("tiny-qwen3")
    assert sum(p.numel() for p in m.parameters()) == cfg.num_params()
    assert llama_config("tiny-qwen3", qk_norm=False).num_params() == cfg.num_params() - 2 * 2 * 64
    assert not any("q_norm" in n for n, _ in build_llama("tiny").named_parameters())


# ---------------------------------------------------------------------------------------------------------------------
# HF interop
# ---------------------------------------------------------------------------------------------------------------------
_GEOM = dict(vocab_size=160, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
             num_key_value_heads=2, head_dim=32, max_position_embeddings=64)


def _hf_qwen3(moe=False):
    transformers = pytest.importorskip("transformers")
    if moe:
        cfg = transformers.Qwen3MoeConfig(**_GEOM, moe_intermediate_size=32, num_experts=8, num_experts_per_tok=2,
                                          norm_topk_prob=True, rope_theta=1e6, rms_norm_eps=1e-6,
                                          attn_implementation="eager")
        cls = transformers.Qwen3MoeForCausalLM
    else:
        cfg = transformers.Qwen3Config(**_GEOM, rope_theta=1e6, rms_norm_eps=1e-6, tie_word_embeddings=True,
                                       attn_implementation="eager")
        cls = transformers.Qwen3ForCausalLM
    torch.manual_seed(0)
    model = cls(cfg)
    with torch.no_grad():   # non-trivial norm weights, so q_norm / k_norm must be loaded to match
        for n, p in model.named_parameters():
            if n.endswith("norm.weight"):
                p.add_(0.2 * torch.randn_like(p))
    return model


@pytest.mark.parametrize("moe", [False, True])
def test_native_qwen3_loads_hf_checkpoint(moe):
    from torchacc_b200.models import build_llama
    hf = _hf_qwen3(moe)
    over = dict(moe_intermediate_size=32, router_aux_loss_coef=0.0) if moe else {}
    native = build_llama("tiny-qwen3-moe" if moe else "tiny-qwen3", **{**_GEOM, **over})
    native.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, 160, (2, 24), generator=torch.Generator().manual_seed(3))
    ref = hf(input_ids=ids, labels=ids)
    out = native(ids, labels=ids, return_logits=True)
    assert abs(float(out["loss"]) - float(ref.loss)) < 1e-4
    assert torch.allclose(out["logits"], ref.logits, atol=1e-4)
    sd, back = hf.state_dict(), native.to_hf_state_dict()
    assert set(back) == set(sd)
    assert all(torch.equal(back[k], sd[k]) for k in sd)


@pytest.fixture
def restore_qwen3_classes():
    transformers = pytest.importorskip("transformers")
    from transformers.models.qwen3 import modeling_qwen3 as mq
    saved = [(c, c.forward) for c in (mq.Qwen3RMSNorm, mq.Qwen3MLP, mq.Qwen3ForCausalLM)]
    rope = mq.apply_rotary_pos_emb
    yield
    for c, f in saved:
        c.forward = f
        if hasattr(c, "_tb_lce_patched"):
            del c._tb_lce_patched
    mq.apply_rotary_pos_emb = rope
    from torchacc_b200.utils.patch import unpatch_all
    unpatch_all()


def test_qwen3_patches_preserve_loss_and_grads(restore_qwen3_classes):
    import torchacc_b200 as ta
    from transformers.models.qwen3 import modeling_qwen3 as mq
    model = _hf_qwen3()
    ids = torch.randint(0, 160, (2, 24), generator=torch.Generator().manual_seed(3))
    ref = model(input_ids=ids, labels=ids)
    ref.loss.backward()
    ref_grads = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    ta.ops.apply_liger_kernel_to_qwen3()
    from torchacc_b200.ops.liger import rms_forward
    assert mq.Qwen3RMSNorm.forward is rms_forward and mq.Qwen3ForCausalLM._tb_lce_patched
    out = model(input_ids=ids, labels=ids)
    assert out.logits is None
    assert abs(float(out.loss) - float(ref.loss)) < 1e-4
    out.loss.backward()
    for n, p in model.named_parameters():
        assert torch.allclose(p.grad, ref_grads[n], atol=2e-5, rtol=1e-3), n
    assert model(input_ids=ids).logits.shape == (2, 24, 160)


def test_hf_family_dispatch_picks_qwen3_only_for_qwen3(monkeypatch):
    transformers = pytest.importorskip("transformers")
    from torchacc_b200.ops import liger
    called = []
    for name in ("apply_liger_kernel_to_qwen3", "apply_liger_kernel_to_qwen3_moe", "apply_liger_kernel_to_qwen2",
                 "apply_liger_kernel_to_llama"):
        monkeypatch.setattr(liger, name, lambda *a, _n=name, **kw: called.append(_n))
    monkeypatch.setattr("torchacc_b200.utils.patch.patch_fa", lambda: None)
    liger.apply_liger_kernel(_hf_qwen3())
    assert called == ["apply_liger_kernel_to_qwen3"]
    called.clear()
    liger.apply_liger_kernel(_hf_qwen3(moe=True))
    assert called == ["apply_liger_kernel_to_qwen3_moe"]
    called.clear()
    cfg = transformers.Qwen2Config(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                   num_attention_heads=2, num_key_value_heads=1)
    liger.apply_liger_kernel(transformers.Qwen2ForCausalLM(cfg))
    assert called == ["apply_liger_kernel_to_qwen2"]


# ---------------------------------------------------------------------------------------------------------------------
# parallel engines (gloo), in the pattern of test_dist_cpu.py
# ---------------------------------------------------------------------------------------------------------------------
_NORMS = ["model.layers.0.self_attn.q_norm.weight", "model.layers.1.self_attn.k_norm.weight"]


def _tiny_qwen3():
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    m = build_llama("tiny-qwen3", hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                    num_key_value_heads=2, head_dim=16, vocab_size=128, max_position_embeddings=128,
                    tie_word_embeddings=False)   # the vocab-parallel lm_head cannot be tied
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(("q_norm.weight", "k_norm.weight")):
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return m


def _data(B=2, S=32, seed=1):
    return torch.randint(0, 128, (B, S), generator=torch.Generator().manual_seed(seed))


def _reference(ids):
    m = _tiny_qwen3()
    out = m(ids, labels=ids)
    out["loss"].backward()
    return float(out["loss"]), {n: p.grad.clone() for n, p in m.named_parameters()}


def _engine_grads(model):
    meta = model._inner_engine_module().get_shard_metadata()
    grads = {}
    for u, g in zip(meta["units"], model.engine.grads()):
        for p in u["params"]:
            grads[(u["prefix"] + "." if u["prefix"] else "") + p["fqn"]] = \
                g[p["offset"]:p["offset"] + p["numel"]].view(p["shape"])
    return grads


def _tp_worker(rank, world, sequence_parallel):
    import torchacc_b200 as ta
    ids = _data()
    ref_loss, ref_grads = _reference(ids)
    cfg = ta.Config()
    cfg.dist.tp.size = 2
    cfg.dist.tp.sequence_parallel = sequence_parallel
    model = ta.accelerate(_tiny_qwen3(), config=cfg)
    out = model(ids, labels=ids)
    assert abs(float(out["loss"]) - ref_loss) < 1e-4, (float(out["loss"]), ref_loss)
    out["loss"].backward()
    grads = _engine_grads(model)
    for n in _NORMS + ["model.layers.0.input_layernorm.weight"]:
        assert torch.allclose(grads[n], ref_grads[n], atol=1e-5, rtol=1e-4), (n, grads[n], ref_grads[n])
    n = "model.layers.1.self_attn.o_proj.weight"
    cols = ref_grads[n].shape[1] // world
    assert torch.allclose(grads[n], ref_grads[n][:, rank * cols:(rank + 1) * cols], atol=1e-5, rtol=1e-4), n
    # the backward ends in all-reduces on the tensor-parallel group (the q / k norm weights among them): both ranks
    # drain that group before the harness tears the process groups down
    import torch.distributed as dist
    core = next(m for m in model.modules() if hasattr(m, "pctx"))
    dist.barrier(group=core.pctx.tp_group)


@pytest.mark.parametrize("sp", [True, False])
def test_qwen3_tensor_parallel_matches_single_process(sp):
    run_distributed(_tp_worker, 2, args=(sp,))


def _cp_worker(rank, world, mode):
    import torch.distributed as dist
    import torchacc_b200 as ta
    from test_dist_cpu import _assert_engine_grads_match
    ids = _data()
    ref_loss, ref_grads = _reference(ids)
    cfg = ta.Config()
    cfg.dist.sp.size = 2
    cfg.dist.sp.mode = mode
    model = ta.accelerate(_tiny_qwen3(), config=cfg)
    out = model(ids, labels=ids)
    loss = out["loss"].detach().clone()
    dist.all_reduce(loss)
    assert abs(float(loss) / world - ref_loss) < 2e-2, (float(loss) / world, ref_loss)
    out["loss"].backward()
    _assert_engine_grads_match(model, ref_grads)
    grads = _engine_grads(model)
    for n in _NORMS:
        assert torch.allclose(grads[n], ref_grads[n], atol=2e-5, rtol=1e-4), (n, grads[n], ref_grads[n])


@pytest.mark.parametrize("mode", ["ulysses", "ring"])
def test_qwen3_context_parallel_matches_single_process(mode):
    run_distributed(_cp_worker, 2, args=(mode,))
