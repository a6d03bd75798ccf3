"""Mixture-of-experts plumbing without a GPU: the PyTorch reference path, the config / presets, HF family dispatch and
the tensor-parallel guard."""
import pytest
import torch
import torch.nn.functional as F


def _naive(x, ids, w, wgu, wd):
    out = torch.zeros_like(x)
    Fd = wgu.shape[1] // 2
    for t in range(x.shape[0]):
        for j in range(ids.shape[1]):
            e = int(ids[t, j])
            gu = wgu[e] @ x[t]
            out[t] += w[t, j] * (wd[e] @ (F.silu(gu[:Fd]) * gu[Fd:]))
    return out


def test_reference_matches_naive_loop():
    from torchacc_b200.ops.moe import moe_experts, moe_router
    g = torch.Generator().manual_seed(0)
    T, H, Fd, E, k = 24, 16, 8, 4, 2
    x = torch.randn(T, H, generator=g)
    w, ids = moe_router(torch.randn(T, E, generator=g), k, True)
    assert torch.allclose(w.sum(-1), torch.ones(T))
    wgu = torch.randn(E, 2 * Fd, H, generator=g)
    wd = torch.randn(E, H, Fd, generator=g)
    res = torch.randn(T, H, generator=g)
    out = moe_experts(x, ids, w, wgu, wd, residual=res)
    assert torch.allclose(out, _naive(x, ids, w, wgu, wd) + res, atol=1e-4, rtol=1e-4)


def test_capacity_bounds_the_padded_layout():
    from torchacc_b200.ops.moe import capacity
    assert capacity(8192, 2, 8) % 128 == 0 and capacity(8192, 2, 8) >= 8192 * 2 + 8 * 127
    assert capacity(1, 1, 1) == 128


def test_config_and_presets():
    from torchacc_b200.models.llama import LlamaConfig, llama_config
    dense = LlamaConfig()
    assert dense.num_experts == 0
    mix = llama_config("mixtral-8x7b")
    assert (mix.num_experts, mix.num_experts_per_tok, mix.moe_intermediate_size) == (8, 2, 14336)
    # Mixtral-8x7B: about 12.9B active parameters per token
    assert 12.5e9 < mix.num_params() < 13.3e9
    tiny = llama_config("tiny-moe")
    assert tiny.num_experts > 0
    assert tiny.flops_per_token(128) < llama_config("tiny-moe", num_experts_per_tok=4).flops_per_token(128)


def test_tiny_moe_model_parameter_names_and_aux_loss():
    from torchacc_b200.models import build_llama
    from torchacc_b200.ops.moe import MoEMLP
    torch.manual_seed(0)
    m = build_llama("tiny-moe", router_aux_loss_coef=0.01)
    assert isinstance(m.model.layers[0].mlp, MoEMLP)
    names = {n for n, _ in m.named_parameters()}
    for n in ("model.layers.0.mlp.gate.weight", "model.layers.0.mlp.experts.gate_up_proj",
              "model.layers.0.mlp.experts.down_proj"):
        assert n in names
    ids = torch.randint(0, 512, (2, 16))
    out = m(input_ids=ids, labels=ids)
    assert "aux_loss" in out and float(out["aux_loss"]) > 0
    out["loss"].backward()
    assert m.model.layers[0].mlp.gate.weight.grad is not None
    assert m.model.layers[0].mlp.experts.gate_up_proj.grad is not None


def test_tensor_parallel_moe_raises():
    from torchacc_b200.models import build_llama
    from torchacc_b200.parallel.tp import shard_llama_for_tp

    class _TP:
        size, rank, group, sequence_parallel = 2, 0, None, False

    with pytest.raises(NotImplementedError):
        shard_llama_for_tp(build_llama("tiny-moe"), _TP())


def test_hf_family_dispatch(monkeypatch):
    pytest.importorskip("transformers")
    import transformers
    from torchacc_b200.ops import liger
    called = []
    for name in ("apply_liger_kernel_to_mixtral", "apply_liger_kernel_to_qwen3_moe", "apply_liger_kernel_to_llama"):
        monkeypatch.setattr(liger, name, lambda *a, _n=name, **kw: called.append(_n))
    monkeypatch.setattr("torchacc_b200.utils.patch.patch_fa", lambda: called.append("patch_fa"))
    cfg = transformers.MixtralConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                     num_attention_heads=2, num_key_value_heads=1, num_local_experts=4)
    liger.apply_liger_kernel(transformers.MixtralForCausalLM(cfg))
    assert "apply_liger_kernel_to_mixtral" in called and "patch_fa" in called
    assert "apply_liger_kernel_to_llama" not in called and "apply_liger_kernel_to_qwen3_moe" not in called


def test_experts_patch_keeps_cpu_on_hf_forward():
    transformers = pytest.importorskip("transformers")
    from transformers.models.mixtral import modeling_mixtral as mm
    from torchacc_b200.ops import liger
    cls = mm.MixtralExperts
    saved = dict(cls.__dict__)
    try:
        cfg = transformers.MixtralConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                         num_attention_heads=2, num_key_value_heads=1, num_local_experts=4)
        ex = cls(cfg)
        torch.nn.init.normal_(ex.gate_up_proj)
        torch.nn.init.normal_(ex.down_proj)
        x = torch.randn(6, 32)
        ids = torch.tensor([[0, 1], [2, 3], [1, 0], [3, 3], [0, 2], [1, 2]])
        w = torch.rand(6, 2)
        ref = ex(x, ids, w)
        liger._patch_experts(mm, "Mixtral")
        assert cls.forward is liger.experts_forward
        assert torch.allclose(ex(x, ids, w), ref)
    finally:
        cls.forward = saved["forward"]
        if "_tb_orig_forward" in cls.__dict__:
            del cls._tb_orig_forward


@pytest.fixture
def restore_moe_classes():
    """Class-level patches are process-global: put every patched HF forward back after the test."""
    import importlib
    saved = []
    for mod in ("transformers.models.mixtral.modeling_mixtral", "transformers.models.qwen3_moe.modeling_qwen3_moe"):
        m = importlib.import_module(mod)
        for cls in vars(m).values():
            if isinstance(cls, type) and cls.__module__ == m.__name__:
                saved.append((cls, dict(cls.__dict__)))
    yield
    for cls, d in saved:
        for attr in ("forward", "_tb_orig_forward", "_tb_lce_patched"):
            if attr in d:
                setattr(cls, attr, d[attr])
            elif attr in cls.__dict__:
                delattr(cls, attr)


@pytest.mark.parametrize("family", ["mixtral", "qwen3_moe"])
def test_moe_family_fused_loss_keeps_hf_aux_loss(family, restore_moe_classes):
    """With output_router_logits the patched causal-LM forward still adds HF's load-balancing loss and returns it."""
    transformers = pytest.importorskip("transformers")
    from torchacc_b200.ops import liger
    torch.manual_seed(0)
    common = dict(vocab_size=160, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                  num_experts_per_tok=2, output_router_logits=True, router_aux_loss_coef=0.5)
    if family == "mixtral":
        model = transformers.MixtralForCausalLM(transformers.MixtralConfig(intermediate_size=96, num_local_experts=4,
                                                                           **common))
        patch = liger.apply_liger_kernel_to_mixtral
    else:
        model = transformers.Qwen3MoeForCausalLM(transformers.Qwen3MoeConfig(
            intermediate_size=96, moe_intermediate_size=48, num_experts=4, **common))
        patch = liger.apply_liger_kernel_to_qwen3_moe
    ids = torch.randint(0, 160, (2, 24), generator=torch.Generator().manual_seed(3))
    ref = model(input_ids=ids, labels=ids)
    assert float(ref.aux_loss) > 0
    ref.loss.backward()
    ref_grads = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    patch()
    out = model(input_ids=ids, labels=ids)
    assert out.logits is None and out.router_logits is not None
    assert abs(float(out.aux_loss) - float(ref.aux_loss)) < 1e-5
    assert abs(float(out.loss) - float(ref.loss)) < 1e-4
    out.loss.backward()
    for n, p in model.named_parameters():
        assert torch.allclose(p.grad, ref_grads[n], atol=2e-5, rtol=1e-3), n


def test_native_aux_loss_is_hfs_load_balancing_loss():
    """Same definition and scale as HF Mixtral's load_balancing_loss_func (so Mixtral's coefficient carries over)."""
    pytest.importorskip("transformers")
    from transformers.models.mixtral.modeling_mixtral import load_balancing_loss_func
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    m = build_llama("tiny-moe", router_aux_loss_coef=0.02)
    ids = torch.randint(0, 512, (2, 16))
    out = m(input_ids=ids, labels=ids)
    logits = tuple(l.mlp.last_router_logits for l in m.model.layers)
    ref = load_balancing_loss_func(logits, m.config.num_experts, m.config.num_experts_per_tok)
    assert torch.allclose(out["aux_loss"], ref, atol=1e-6, rtol=1e-5)
