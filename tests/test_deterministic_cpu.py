"""Deterministic mode plumbing (no GPU): the config field, the process switches set by accelerate(), the HF
flash-attention replacement forwarding ``deterministic`` and ring attention's one-time warning."""
import json

import pytest
import torch

import torchacc_b200 as ta
from torchacc_b200.config import ComputeConfig, Config, ConfigError


def test_config_field_default_validation_and_round_trip():
    cfg = Config()
    assert cfg.compute.deterministic is False
    cfg.compute.deterministic = 1
    with pytest.raises(ConfigError):
        cfg.validate()
    cfg.compute.deterministic = True
    cfg.validate()
    d = cfg.compute.to_dict()
    assert d["deterministic"] is True
    back = ComputeConfig.from_dict(json.loads(json.dumps(d)))
    assert back.deterministic is True and back == cfg.compute
    assert ComputeConfig.from_dict({}).deterministic is False


def test_accelerate_sets_and_clears_the_process_switch():
    from torchacc_b200.ops import attention as A
    from torchacc_b200.ops import optim as O
    try:
        cfg = Config()
        cfg.compute.deterministic = True
        ta.accelerate(torch.nn.Linear(4, 4), config=cfg)
        assert A._DETERMINISTIC and O._DETERMINISTIC
        assert A.deterministic_enabled() and O.deterministic_enabled()
        ta.accelerate(torch.nn.Linear(4, 4), config=Config())
        assert not A._DETERMINISTIC and not O._DETERMINISTIC
        assert A.deterministic_enabled() == torch.are_deterministic_algorithms_enabled()
    finally:
        A.set_deterministic(False)
        O.set_deterministic(False)


def test_effective_flag_honours_the_call_and_torch_global():
    from torchacc_b200.ops import attention as A
    from torchacc_b200.ops import optim as O
    assert not A.deterministic_enabled()
    assert A.deterministic_enabled(True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert A.deterministic_enabled() and O.deterministic_enabled()
    finally:
        torch.use_deterministic_algorithms(prev)


def _record_attention_calls(monkeypatch):
    from torchacc_b200.ops import attention as A
    calls = []

    def rec(name):
        def fn(q, *args, **kwargs):
            calls.append((name, kwargs.get("deterministic")))
            return q
        return fn

    monkeypatch.setattr(A, "flash_attn_func", rec("fixed"))
    monkeypatch.setattr(A, "flash_attn_varlen_func", rec("varlen"))
    monkeypatch.setattr(A, "flash_attn_varlen_position_ids_func", rec("position_ids"))
    return calls


def test_hf_flash_attention_forward_forwards_deterministic(monkeypatch):
    from torchacc_b200.utils.patch import _hf_flash_attention_forward
    calls = _record_attention_calls(monkeypatch)
    monkeypatch.delenv("FLASH_ATTENTION_DETERMINISTIC", raising=False)
    q = torch.zeros(2, 8, 2, 16)
    _hf_flash_attention_forward(q, q, q, deterministic=True)
    _hf_flash_attention_forward(q, q, q, deterministic=False)
    _hf_flash_attention_forward(q, q, q)
    mask = torch.ones(2, 8, dtype=torch.int32)
    mask[1, 5:] = 0
    _hf_flash_attention_forward(q, q, q, attention_mask=mask, deterministic=True)
    pos = torch.cat([torch.arange(4), torch.arange(4)])[None]
    _hf_flash_attention_forward(q[:1], q[:1], q[:1], position_ids=pos, deterministic=True)
    assert calls == [("fixed", True), ("fixed", False), ("fixed", False), ("varlen", True), ("position_ids", True)]


def test_hf_flash_attention_forward_honours_the_env_var(monkeypatch):
    from torchacc_b200.utils.patch import _hf_flash_attention_forward
    calls = _record_attention_calls(monkeypatch)
    q = torch.zeros(1, 8, 2, 16)
    monkeypatch.setenv("FLASH_ATTENTION_DETERMINISTIC", "1")
    _hf_flash_attention_forward(q, q, q)
    _hf_flash_attention_forward(q, q, q, deterministic=False)     # an explicit argument wins
    monkeypatch.setenv("FLASH_ATTENTION_DETERMINISTIC", "0")
    _hf_flash_attention_forward(q, q, q)
    assert calls == [("fixed", True), ("fixed", False), ("fixed", False)]


def test_ring_attention_warns_once_that_it_is_not_deterministic(monkeypatch):
    from torchacc_b200.ops import attention as A
    from torchacc_b200.ops.context_parallel import ring as R
    warnings = []

    class _Log:
        def warning(self, msg, *args):
            warnings.append(msg % args if args else msg)

    monkeypatch.setattr(A, "logger", _Log())
    monkeypatch.setattr(A, "_warned", set())
    monkeypatch.setattr(R._RingAttnFn, "apply", staticmethod(lambda q, *args: q))
    q = torch.zeros(1, 8, 2, 16)
    R.ring_attention(q, q, q, deterministic=False)
    assert warnings == []
    for _ in range(3):
        R.ring_attention(q, q, q, deterministic=True)
    assert len(warnings) == 1 and "deterministic" in warnings[0]
