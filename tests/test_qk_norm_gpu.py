"""Qwen3 on the GPU: the fused per-head QK-RMSNorm + RoPE kernels (csrc/ops/norm_rope_act.cu) against an fp64 reference
of their arithmetic contract, the native tiny-qwen3 / tiny-qwen3-moe against the fp32 CPU model, training through the
FSDP engine (also bitwise reproducible), and HF Qwen3ForCausalLM through accelerate().

Contract, per q / k head row in fp32: rstd = rsqrt(mean(x^2) + eps), z = x rstd w, out = rope(z), one rounding at the
end; V copied.  Backward: u = rope^-1(g), xhat = x rstd, dx = rstd (u w - xhat mean(u w xhat)), dw = sum u xhat.
Tolerances are ulps of the output dtype (``check`` of test_ops_kernels_gpu) plus derived floors."""
import functools

import pytest
import torch

from test_ops_kernels_gpu import check

pytestmark = pytest.mark.gpu

DEV = "cuda"
MAX_POS = 131072
EPS = 1e-6


@functools.lru_cache(maxsize=None)
def _tables(D):
    from torchacc_b200.ops.rope import rope_tables
    return rope_tables(MAX_POS, D, theta=1e6, device=DEV)


def _inputs(T, hq, hk, D, dtype, gen):
    x = torch.randn(T, hq + 2 * hk, D, device=DEV, generator=gen)
    x[0, :hq + hk] = 0.0                                                                   # all-zero rows
    x[1, :hq + hk] = 3.0e4 * torch.sign(torch.randn(hq + hk, D, device=DEV, generator=gen))  # +-3e4 (fp16-safe)
    x[2, :hq + hk] *= 1e-2
    x[2, :hq + hk, D // 3] = 1.0e3                                                         # one dominant element
    return x.reshape(T, -1).to(dtype)


def _positions(T, B, pos_mode, gen):
    if pos_mode == "seq":
        return None, T // B, torch.arange(T, device=DEV) % (T // B)
    pos = torch.randint(0, MAX_POS, (T,), device=DEV, generator=gen, dtype=torch.int32)
    pos[0], pos[-1], pos[T // 2] = MAX_POS - 1, 0, MAX_POS - 1                          # the table's last row, and its first
    return pos, MAX_POS, pos.long()


def _rope64(a, b, c, s):
    """(a, b) halves rotated by (c, s); also the no-cancellation magnitude of each output."""
    return (torch.cat([a * c - b * s, b * c + a * s], -1),
            torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], -1))


def _run(D, dtype, heads, pos_mode, B, S, seed=0):
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import qk_norm_rope_qkv
    hq, hk = heads
    hqk, T, half = hq + hk, B * S, D // 2
    gen = torch.Generator(device=DEV).manual_seed(seed + D + hq)
    cos, sin = _tables(D)
    positions, seq_len, pos_long = _positions(T, B, pos_mode, gen)
    qkv = _inputs(T, hq, hk, D, dtype, gen).requires_grad_()
    wq = (1 + 0.1 * torch.randn(D, device=DEV, generator=gen)).to(dtype).requires_grad_()
    wk = (1 + 0.1 * torch.randn(D, device=DEV, generator=gen)).to(dtype).requires_grad_()
    gout = torch.randn(T, (hq + 2 * hk) * D, device=DEV, generator=gen).to(dtype)
    before = qkv.detach().clone()
    n0 = nat.LAUNCHES
    out = qk_norm_rope_qkv(qkv, hq, hk, D, wq, wk, EPS, cos, sin, positions, seq_len)
    out.backward(gout, retain_graph=True)
    assert nat.LAUNCHES - n0 == 2, "forward and backward are one kernel each"
    tag = f"qk_norm_rope D={D} {dtype} {hq}/{hk} {pos_mode} T={T}"
    assert torch.equal(qkv.detach(), before), f"{tag}: the input was modified"

    x64 = before.double().view(T, hq + 2 * hk, D)[:, :hqk]
    w64 = torch.cat([wq.detach().double().expand(hq, D), wk.detach().double().expand(hk, D)], 0)
    c64, s64 = cos[pos_long].double().unsqueeze(1), sin[pos_long].double().unsqueeze(1)
    rs64 = torch.rsqrt(x64.square().mean(-1, keepdim=True) + EPS)
    xh = x64 * rs64
    z = xh * w64
    ref, mag = _rope64(z[..., :half], z[..., half:], c64, s64)
    # z carries the fp32 error of the sum of squares (<= 16 sequential adds per lane + 4 shuffle adds, relative
    # <= 20 x 2^-24), rsqrtf (2 ulp) and two products: < 2^-19 relative.  The rotation adds 2^-23 per product before
    # the one rounding: floor 2^-18 x (|za c| + |zb s|), which only matters where the two products cancel.
    o = out.detach().view(T, hq + 2 * hk, D)
    check(o[:, :hq], ref[:, :hq], f"{tag} q", floor=2.0 ** -18 * mag[:, :hq])
    check(o[:, hq:hqk], ref[:, hq:], f"{tag} k", floor=2.0 ** -18 * mag[:, hq:])
    assert torch.equal(o[:, hqk:], before.view(T, hq + 2 * hk, D)[:, hqk:]), f"{tag}: V is not a bitwise copy"

    g64 = gout.double().view(T, hq + 2 * hk, D)[:, :hqk]
    g1, g2 = g64[..., :half], g64[..., half:]
    u, umag = _rope64(g1, g2, c64, -s64)
    dot = (u * w64 * xh).mean(-1, keepdim=True)
    dx64 = rs64 * (u * w64 - xh * dot)
    # u has error <= 2^-23 (|g1 c| + |g2 s|) (umag), xhat <= 2^-19 relative, the mean is an fp32 sum of D terms (<= 20
    # sequential adds per lane, 2^-19 relative of sum |u w xhat| / D), and dx cancels two terms: floor 2^-17 x the row's
    # largest rstd (umag |w| + |xhat dot|-scale term), computed without cancellation.
    scale_row = (rs64 * (umag * w64.abs() + (xh * (u * w64 * xh).abs().mean(-1, keepdim=True)).abs())) \
        .amax(-1, keepdim=True)
    dq = qkv.grad.view(T, hq + 2 * hk, D)
    check(dq[:, :hq], dx64[:, :hq], f"{tag} dq", floor=2.0 ** -17 * scale_row[:, :hq])
    check(dq[:, hq:hqk], dx64[:, hq:], f"{tag} dk", floor=2.0 ** -17 * scale_row[:, hq:])
    assert torch.equal(dq[:, hqk:], gout.view(T, hq + 2 * hk, D)[:, hqk:]), f"{tag}: dV is not the incoming gradient"

    # dw: each lane sums its rows in fp32 (at most ceil(rows / (CTAs x rows per CTA)) of them), the CTA sums its groups
    # in thread order (256 / G), the host sums the CTAs' partials: a product passes through n sequential fp32 adds,
    # error <= n 2^-24 of sum |u xhat|, plus the 2^-18 relative error of u xhat itself, then one rounding to the dtype
    G = 1 << max(0, (D // 16 - 1).bit_length())
    rows_per_cta = 256 // G
    rows = T * (hq + 2 * hk)
    ctas = max(1, min(nat.num_sms() * 2, -(-rows // rows_per_cta)))
    n_adds = -(-rows // (ctas * rows_per_cta)) + rows_per_cta + ctas
    p = u * xh
    for name, w, sl in (("dq_weight", wq, slice(0, hq)), ("dk_weight", wk, slice(hq, hqk))):
        ref_w = p[:, sl].sum((0, 1))
        floor = (n_adds * 2.0 ** -24 + 2.0 ** -18) * p[:, sl].abs().sum((0, 1))
        check(w.grad, ref_w, f"{tag} {name}", floor=floor)

    # the backward again on the same graph: bitwise the same dqkv and weight gradients (no atomics)
    first = [qkv.grad.clone(), wq.grad.clone(), wk.grad.clone()]
    qkv.grad = wq.grad = wk.grad = None
    out.backward(gout)
    for a, b, n in zip(first, [qkv.grad, wq.grad, wk.grad], ("dqkv", "dq_weight", "dk_weight")):
        assert torch.equal(a, b), f"{tag}: {n} differs between two identical backward passes"


@pytest.mark.parametrize("pos_mode", ["seq", "positions"])
@pytest.mark.parametrize("heads", [(32, 8), (16, 8), (8, 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_qk_norm_rope_matches_fp64(D, dtype, heads, pos_mode):
    _run(D, dtype, heads, pos_mode, B=3, S=97)


def test_qk_norm_rope_grid_stride_loop():
    """T = 8192 with 40 q + k heads (the Qwen3-8B layer): 8192 x 48 head rows / 32 rows per CTA is far more than the
    forward's 8 CTAs per SM and the backward's 2, so both kernels loop over rows."""
    _run(128, torch.bfloat16, (32, 8), "positions", B=2, S=4096)


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _tiny(name, device, dtype):
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    with torch.device(device):
        m = build_llama(name, hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, head_dim=128, vocab_size=2048, max_position_embeddings=512, dtype=dtype)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(("q_norm.weight", "k_norm.weight")):
                p.add_((0.2 * torch.randn(p.shape, generator=g)).to(device, dtype))
    return m


@pytest.mark.parametrize("name", ["tiny-qwen3", "tiny-qwen3-moe"])
def test_qwen3_native_matches_fp32_reference(name):
    dev = torch.device("cuda", 0)
    ref = _tiny(name, "cpu", torch.float32)
    nat_model = _tiny(name, dev, torch.bfloat16)
    nat_model.load_state_dict({k: v.to(dev, torch.bfloat16) for k, v in ref.state_dict().items()})
    ids = torch.randint(0, 2048, (2, 256))
    out_r = ref(ids, labels=ids)
    out_n = nat_model(ids.to(dev), labels=ids.to(dev))
    assert abs(float(out_r["loss"]) - float(out_n["loss"])) < 3e-2, (float(out_r["loss"]), float(out_n["loss"]))
    out_r["loss"].backward()
    out_n["loss"].backward()
    # with bf16 router logits about 1 % of the tokens pick a different expert than in fp32 (their near-uniform
    # softmax at init leaves ties within bf16 rounding), and each such token changes its whole expert-branch gradient:
    # the MoE model's bound is looser than the dense model's
    bound = 2.5e-1 if "moe" in name else 8e-2
    for (n, pr), (_, pn) in zip(ref.named_parameters(), nat_model.named_parameters()):
        g_r, g_n = pr.grad.float(), pn.grad.float().cpu()
        rel = (g_r - g_n).norm().item() / (g_r.norm().item() + 1e-6)
        print(f"[grad] {name} {n}: relative error {rel:.4f}")
        assert rel < bound, f"{n}: relative grad error {rel:.3f}"


def _train(steps, deterministic=False):
    import torchacc_b200 as ta
    model = _tiny("tiny-qwen3", "cuda", torch.bfloat16)
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.compute.deterministic = deterministic
    cfg.memory.gc = True
    cfg.memory.gc_cls = {"LlamaDecoderLayer"}
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=2e-3)
    ids = torch.randint(0, 2048, (4, 128), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    losses = []
    for _ in range(steps):
        out = model(input_ids=ids, labels=ids)
        out["loss"].backward()
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        losses.append(out["loss"].detach().clone())
    torch.cuda.synchronize()
    return model, losses, [p.detach().clone() for p in model.parameters()]


def test_qwen3_engine_trains_on_native_kernels():
    from torchacc_b200 import _native as nat
    n0 = nat.LAUNCHES
    model, losses, _ = _train(8)
    assert nat.LAUNCHES > n0
    assert float(losses[-1]) < float(losses[0]) - 0.5, losses
    assert model.engine.stats.get("wgrad_fallbacks", 0) == 0, model.engine.stats


def test_qwen3_training_is_bitwise_reproducible(monkeypatch):
    from torchacc_b200.ops import attention as A, optim as O
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        (_, la, pa), (_, lb, pb) = _train(2, True), _train(2, True)
    finally:
        torch.use_deterministic_algorithms(prev)
        A.set_deterministic(False)
        O.set_deterministic(False)
    for i, (x, y) in enumerate(zip(la, lb)):
        assert torch.equal(x, y), f"step {i}: loss {float(x)!r} vs {float(y)!r}"
    for i, (x, y) in enumerate(zip(pa, pb)):
        assert torch.equal(x, y), f"parameter {i}: max diff {float((x.float() - y.float()).abs().max()):.3g}"


def test_hf_qwen3_through_accelerate():
    """accelerate(HF Qwen3ForCausalLM): patched classes, native RoPE and attention launches, loss close to stock HF, and
    training proceeds."""
    import copy
    transformers = pytest.importorskip("transformers")
    import torchacc_b200 as ta
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops.liger import rms_forward
    from torchacc_b200.utils.patch import unpatch_all
    from transformers.models.qwen3 import modeling_qwen3 as mq
    dev = torch.device("cuda", 0)
    cfg = transformers.Qwen3Config(vocab_size=2048, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                                   num_attention_heads=8, num_key_value_heads=2, head_dim=128,
                                   max_position_embeddings=512, rms_norm_eps=1e-6, tie_word_embeddings=False,
                                   attn_implementation="sdpa", use_cache=False)
    torch.manual_seed(0)
    ref = transformers.Qwen3ForCausalLM(cfg).to(dev, torch.bfloat16)
    ours = copy.deepcopy(ref)
    ids = torch.randint(0, 2048, (2, 256), device=dev)
    ref_loss = ref(input_ids=ids, labels=ids).loss
    saved = [(c, c.forward) for c in (mq.Qwen3RMSNorm, mq.Qwen3MLP, mq.Qwen3ForCausalLM)]
    try:
        ours.config._attn_implementation = "flash_attention_2"       # HF dispatches to the patched interface
        c = ta.Config()
        c.compute.bf16 = True
        c.dist.fsdp.wrap_layer_cls = {"Qwen3DecoderLayer"}
        model = ta.accelerate(ours, config=c)
        assert mq.apply_rotary_pos_emb.__name__ == "hf_apply_rotary_pos_emb"
        assert mq.Qwen3RMSNorm.forward is rms_forward and mq.Qwen3ForCausalLM._tb_lce_patched
        n0 = nat.LAUNCHES
        out = model(input_ids=ids, labels=ids)
        launches = nat.LAUNCHES - n0
        # per layer: 4 projections + 2 layer norms + q_norm + k_norm + 2 RoPE + attention + SwiGLU, plus the final
        # norm and the loss
        assert launches >= 2 * (4 + 2 + 2 + 2 + 1 + 1) + 2, launches
        assert abs(float(out.loss) - float(ref_loss)) < 5e-2, (float(out.loss), float(ref_loss))
        opt = ta.optim.FusedAdamW(model.parameters(), lr=1e-3)   # at 2e-3 the loss of this model oscillates after a few steps
        losses = []
        for _ in range(6):
            l = model(input_ids=ids, labels=ids).loss
            l.backward()
            opt.step()
            opt.zero_grad()
            losses.append(float(l))
        assert losses[-1] < losses[0] - 0.5, losses
    finally:
        for cls, f in saved:
            cls.forward = f
            if hasattr(cls, "_tb_lce_patched"):
                del cls._tb_lce_patched
        unpatch_all()
