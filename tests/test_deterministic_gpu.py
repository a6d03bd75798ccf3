"""Deterministic mode on the GPU: the atomic-free attention dQ kernel (every feature of the native backward, bitwise
repeatable, matching the fp32 reference), the ordered gradient-norm reduction and a bitwise reproducible training run
of the native Llama."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _check(a, b, name, rtol, atol):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = int((err > tol).sum())
    assert bad == 0, f"{name}: {bad}/{a.numel()} off, max err {float(err.max()):.4g} (ref max {float(b.abs().max()):.3g})"


def _mk(g, dtype):
    return lambda *shape: (torch.randn(*shape, device=DEV, generator=g) * 0.8).to(dtype)


@pytest.fixture(autouse=True)
def _native_backend():
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    yield
    A.set_attention_backend("auto")
    A.set_deterministic(False)


ATTN_CASES = [
    # dtype,         B, Sq,  Sk,  Hq, Hk, D,   causal, window,    alibi, dropout
    (torch.bfloat16, 2, 256, 256, 4, 4, 128, False, (-1, -1), False, 0.0),    # non-causal MHA
    (torch.bfloat16, 2, 256, 256, 4, 4, 128, True, (-1, -1), False, 0.0),     # causal
    (torch.bfloat16, 1, 512, 512, 8, 2, 128, True, (-1, -1), False, 0.0),     # GQA
    (torch.bfloat16, 1, 384, 384, 4, 1, 64, True, (-1, -1), False, 0.0),      # MQA, head dim 64
    (torch.bfloat16, 2, 200, 200, 4, 2, 128, True, (-1, -1), False, 0.0),     # ragged tail
    (torch.bfloat16, 1, 130, 390, 4, 4, 128, True, (-1, -1), False, 0.0),     # Sq < Sk, bottom-right causal
    (torch.bfloat16, 1, 390, 130, 4, 2, 64, False, (-1, -1), False, 0.0),     # Sq > Sk, non-causal
    (torch.bfloat16, 1, 640, 640, 4, 2, 128, True, (100, 0), False, 0.0),     # sliding window
    (torch.bfloat16, 1, 512, 512, 2, 2, 128, False, (64, 32), False, 0.0),    # local, non-causal
    (torch.bfloat16, 1, 320, 320, 4, 4, 96, False, (-1, -1), False, 0.0),     # head dim 96 (padded to 128)
    (torch.float16, 2, 256, 256, 4, 4, 128, True, (-1, -1), False, 0.0),      # fp16
    (torch.float16, 1, 384, 384, 8, 2, 64, False, (-1, -1), False, 0.0),      # fp16, head dim 64
    (torch.bfloat16, 2, 256, 256, 4, 4, 128, True, (-1, -1), True, 0.0),      # ALiBi
    (torch.float16, 1, 200, 328, 4, 1, 128, True, (64, 0), True, 0.0),        # ALiBi + window + fp16 + MQA
    (torch.bfloat16, 2, 256, 256, 4, 2, 128, True, (-1, -1), False, 0.17),    # dropout
    (torch.bfloat16, 1, 200, 328, 4, 4, 64, False, (-1, -1), False, 0.1),     # dropout, ragged, Sq != Sk
]


def _tol(dtype):
    return 3e-2 if dtype == torch.bfloat16 else 6e-3


def _grads(fn, inputs, do):
    leaves = [t.detach().clone().requires_grad_() for t in inputs]
    out = fn(*leaves)
    out.backward(do)
    return [out.detach()] + [t.grad for t in leaves]


def _assert_repeatable(fn, inputs, do, runs=5):
    """`runs` backward passes of fn on the same inputs: bitwise-equal outputs and gradients, each run of the
    deterministic dQ kernel counted.  Returns the first run's (out, *grads)."""
    from torchacc_b200.ops import attention as A
    first = None
    for r in range(runs):
        n0 = A.DETERMINISTIC_BWD_CALLS
        res = _grads(fn, inputs, do)
        assert A.DETERMINISTIC_BWD_CALLS > n0, "the deterministic dQ kernel did not run"
        if first is None:
            first = res
            continue
        for name, a, b in zip(("out", "dq", "dk", "dv"), first, res):
            assert torch.equal(a, b), f"run {r}: {name} differs from run 0 (max {float((a - b).abs().max()):.3g})"
    return first


@pytest.mark.parametrize("dtype,B,Sq,Sk,Hq,Hk,D,causal,window,alibi,p", ATTN_CASES)
def test_deterministic_attention_matches_reference_and_repeats(dtype, B, Sq, Sk, Hq, Hk, D, causal, window, alibi,
                                                               p):
    from torchacc_b200.ops import attention as A
    g = torch.Generator(device=DEV).manual_seed(7)
    mk = _mk(g, dtype)
    q, k, v, do = mk(B, Sq, Hq, D), mk(B, Sk, Hk, D), mk(B, Sk, Hk, D), mk(B, Sq, Hq, D)
    slopes = (torch.rand(B, Hq, device=DEV, generator=g) * 0.3) if alibi else None

    def fn(q_, k_, v_):
        torch.manual_seed(1234)           # dropout seed
        return A.flash_attn_func(q_, k_, v_, dropout_p=p, causal=causal, window_size=window, alibi_slopes=slopes,
                                 deterministic=True)

    out, dq, dk, dv = _assert_repeatable(fn, (q, k, v), do)
    keep = None
    if p > 0:
        torch.manual_seed(1234)
        _, _, keep = A.flash_attn_func(q, k, v, dropout_p=p, causal=causal, return_attn_probs=True)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, _ = A.attention_reference(qf, kf, vf, None, causal, window, slopes, p, keep_mask=keep)
    ref.backward(do.float())
    tol = _tol(dtype)
    _check(out, ref, "out", tol, tol)
    _check(dq, qf.grad, "dq", tol, tol)
    _check(dk, kf.grad, "dk", tol, tol)
    _check(dv, vf.grad, "dv", tol, tol)
    # dK / dV come from the same main kernel with its dQ step compiled out: bitwise equal to the default backward
    # (which has no atomics on dK / dV); dQ agrees within rounding
    outd, dqd, dkd, dvd = _grads(lambda a, b, c: (torch.manual_seed(1234), A.flash_attn_func(
        a, b, c, dropout_p=p, causal=causal, window_size=window, alibi_slopes=slopes))[1], (q, k, v), do)
    assert torch.equal(outd, out) and torch.equal(dkd, dk) and torch.equal(dvd, dv)
    _check(dq, dqd, "dq vs default backward", tol, tol)


@pytest.mark.parametrize("causal", [False, True])
def test_deterministic_varlen_mask(causal):
    from torchacc_b200.ops import attention as A
    B, S, H, Hk, D = 3, 256, 4, 2, 128
    g = torch.Generator(device=DEV).manual_seed(5)
    mk = _mk(g, torch.bfloat16)
    q, k, v, do = mk(B, S, H, D), mk(B, S, Hk, D), mk(B, S, Hk, D), mk(B, S, H, D)
    lens = torch.tensor([256, 100, 177], device=DEV)
    mask = (torch.arange(S, device=DEV)[None, :] < lens[:, None]).int()
    fn = lambda q_, k_, v_: A.flash_attn_varlen_func(q_, k_, v_, mask, causal=causal, deterministic=True)
    out, dq, dk, dv = _assert_repeatable(fn, (q, k, v), do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, _ = A.attention_reference_masked(qf, kf, vf, mask.bool(), 1 / math.sqrt(D), causal, (-1, -1))
    ref.backward(do.float())
    for name, a, b in (("out", out, ref), ("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
        _check(a, b, name, 3e-2, 3e-2)


def test_deterministic_position_ids_packing():
    from torchacc_b200.ops import attention as A
    H, Hk, D = 4, 2, 128
    seqs = [100, 156, 128]
    total = sum(seqs)
    pos = torch.cat([torch.arange(n, device=DEV) for n in seqs])[None]
    g = torch.Generator(device=DEV).manual_seed(8)
    mk = _mk(g, torch.bfloat16)
    q, k, v, do = mk(1, total, H, D), mk(1, total, Hk, D), mk(1, total, Hk, D), mk(1, total, H, D)
    fn = lambda q_, k_, v_: A.flash_attn_varlen_position_ids_func(q_, k_, v_, pos, causal=True, deterministic=True)
    out, dq, dk, dv = _assert_repeatable(fn, (q, k, v), do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    refs, off = [], 0
    for n in seqs:
        r, _ = A.attention_reference(qf[:, off:off + n], kf[:, off:off + n], vf[:, off:off + n], None, True)
        refs.append(r)
        off += n
    ref = torch.cat(refs, 1)
    ref.backward(do.float())
    for name, a, b in (("out", out, ref), ("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
        _check(a, b, name, 3e-2, 3e-2)


def test_qkvpacked_tokens_follows_the_process_switch():
    """The native Llama's fast path has no per-call flag: set_deterministic (what Config.compute.deterministic does)
    makes its dqkv bitwise repeatable."""
    from torchacc_b200.ops import attention as A
    B, S, hq, hk, D = 2, 384, 8, 2, 128
    T = B * S
    g = torch.Generator(device=DEV).manual_seed(0)
    qkv = (torch.randn(T, (hq + 2 * hk) * D, device=DEV, generator=g) * 0.7).bfloat16()
    do = torch.randn(T, hq * D, device=DEV, generator=g).bfloat16()
    A.set_deterministic(True)
    grads = []
    for _ in range(5):
        n0 = A.DETERMINISTIC_BWD_CALLS
        x = qkv.clone().requires_grad_()
        A.flash_attn_qkvpacked_tokens(x, hq, hk, D, B, S, causal=True).backward(do)
        assert A.DETERMINISTIC_BWD_CALLS == n0 + 1
        grads.append(x.grad)
    assert all(torch.equal(grads[0], d) for d in grads[1:])
    x = qkv.float().requires_grad_()
    q = x[:, :hq * D].reshape(B, S, hq, D)
    k = x[:, hq * D:(hq + hk) * D].reshape(B, S, hk, D)
    v = x[:, (hq + hk) * D:].reshape(B, S, hk, D)
    ref, _ = A.attention_reference(q, k, v, None, True)
    ref.reshape(T, hq * D).backward(do.float())
    _check(grads[0], x.grad, "dqkv", 3e-2, 3e-2)
    A.set_deterministic(False)
    n0 = A.DETERMINISTIC_BWD_CALLS
    x = qkv.clone().requires_grad_()
    A.flash_attn_qkvpacked_tokens(x, hq, hk, D, B, S, causal=True).backward(do)
    assert A.DETERMINISTIC_BWD_CALLS == n0, "the default path must stay the default"


def test_ordered_grad_sqnorm_is_bitwise_repeatable():
    from torchacc_b200.ops import optim as O
    g = torch.Generator(device=DEV).manual_seed(3)
    grads = [torch.randn(n, device=DEV, generator=g).to(dt) for n, dt in
             ((3_000_001, torch.bfloat16), (1_234_567, torch.float32), (1000, torch.bfloat16), (7, torch.float32))]
    exact = sum(float((t.double() ** 2).sum()) for t in grads)
    default = O.grad_sqnorm(grads)
    O.set_deterministic(True)
    try:
        outs = [O.grad_sqnorm(grads) for _ in range(5)]
        assert all(torch.equal(outs[0], o) for o in outs[1:])
        assert abs(float(outs[0][0]) - exact) <= 1e-6 * exact, (float(outs[0][0]), exact)
        assert float(outs[0][1]) == 0.0
        assert abs(float(default[0]) - float(outs[0][0])) <= 1e-5 * exact
        # the ticket counter is back at zero after every launch
        assert all(int(c.item()) == 0 for _, c in O._ORDERED_WS.values())
        bad = [t.clone() for t in grads]
        bad[1][12345] = float("inf")
        o_bad = [O.grad_sqnorm(bad) for _ in range(2)]
        assert float(o_bad[0][1]) == 1.0 and torch.equal(o_bad[0], o_bad[1])
        bad[1][12345] = float("nan")
        assert float(O.grad_sqnorm(bad)[1]) == 1.0
        # torch's global switch selects the same path
        O.set_deterministic(False)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            assert torch.equal(O.grad_sqnorm(grads), outs[0])
        finally:
            torch.use_deterministic_algorithms(prev)
    finally:
        O.set_deterministic(False)


def _tiny_llama():
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    with torch.device(DEV):
        return build_llama("tiny", hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=4,
                           num_key_value_heads=2, head_dim=128, vocab_size=2048, max_position_embeddings=512,
                           dtype=torch.bfloat16)


def _train(config_flag: bool):
    import torchacc_b200 as ta
    from torchacc_b200.ops import attention as A
    model = _tiny_llama()
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.compute.deterministic = config_flag
    cfg.memory.gc = True
    cfg.memory.gc_cls = {"LlamaDecoderLayer"}
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=2e-3)
    ids = torch.randint(0, 2048, (4, 256), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    n0 = A.DETERMINISTIC_BWD_CALLS
    losses = []
    for _ in range(4):
        out = model(input_ids=ids, labels=ids)
        out["loss"].backward()
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        losses.append(out["loss"].detach().clone())
    torch.cuda.synchronize()
    assert A.DETERMINISTIC_BWD_CALLS > n0, "the training step did not use the deterministic attention backward"
    return losses, [p.detach().clone() for p in model.parameters()]


def _assert_same_runs(a, b):
    (la, pa), (lb, pb) = a, b
    for i, (x, y) in enumerate(zip(la, lb)):
        assert torch.equal(x, y), f"step {i}: loss {float(x)!r} vs {float(y)!r}"
    assert len(pa) == len(pb)
    for i, (x, y) in enumerate(zip(pa, pb)):
        assert torch.equal(x, y), f"parameter {i}: max diff {float((x.float() - y.float()).abs().max()):.3g}"


def test_training_is_bitwise_reproducible_with_the_config_switch():
    from torchacc_b200.ops import attention as A, optim as O
    try:
        _assert_same_runs(_train(True), _train(True))
    finally:
        A.set_deterministic(False)
        O.set_deterministic(False)


def test_training_is_bitwise_reproducible_with_torch_deterministic_algorithms(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # what torch requires of cuBLAS in this mode
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _assert_same_runs(_train(False), _train(False))
    finally:
        torch.use_deterministic_algorithms(prev)
