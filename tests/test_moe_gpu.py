"""Mixture-of-experts kernels on the GPU: grouped GEMMs, routing kernels, ``moe_experts`` / ``moe_router`` and the native
``tiny-moe`` model."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda", 0)


def _close(a, b, rtol, atol, what=""):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    assert bool((err <= tol).all()), f"{what}: max err {err.max().item():.4g} (max |ref| {b.abs().max().item():.4g})"


def _ids_with_counts(counts, k, device, seed=0):
    """expert_ids [T, k] whose per-expert entry counts are `counts` (each token picks k distinct experts when possible)."""
    g = torch.Generator().manual_seed(seed)
    flat = torch.cat([torch.full((c,), e, dtype=torch.int64) for e, c in enumerate(counts)])
    flat = flat[torch.randperm(flat.numel(), generator=g)]
    assert flat.numel() % k == 0
    return flat.view(-1, k).to(device)


def _index(ids, E):
    from torchacc_b200.ops.moe import MoEIndex
    return MoEIndex(ids, E)


def _sorted_rows(idx, x):
    """x_perm built on the host from the index (rows sorted by expert, zero padding)."""
    xp = torch.zeros((idx.rows, x.shape[1]), dtype=x.dtype, device=x.device)
    pos = idx.pos.long().flatten()
    xp[pos] = x.repeat_interleave(idx.k, 0)
    return xp


COUNT_CASES = {
    "mixed": [0, 1, 127, 128, 129, 300, 5, 2],
    "one_expert": [512, 0, 0, 0],
    "e128": [(i * 37) % 50 for i in range(128)],
    "last_expert": [0] * 63 + [4096],                 # every entry to expert E - 1
    "e256": [(i * 53) % 500 for i in range(256)],     # 62 rounds of 1024 entries, counts up to 498
}


@pytest.mark.parametrize("case", list(COUNT_CASES))
def test_index_build_matches_stable_argsort(case):
    dev = _dev()
    counts = COUNT_CASES[case]
    k = 2
    if sum(counts) % k:
        counts = counts + [1]
    E = len(counts)
    ids = _ids_with_counts(counts, k, dev)
    idx = _index(ids, E)
    torch.cuda.synchronize()
    cnt = torch.bincount(ids.flatten(), minlength=E)
    assert torch.equal(idx.counts.long().cpu(), cnt.cpu())
    padded = (cnt + 127) // 128 * 128
    off = torch.zeros(E + 1, dtype=torch.long, device=dev)
    off[1:] = padded.cumsum(0)
    assert torch.equal(idx.offsets.long(), off)
    tiles = int(off[-1]) // 128
    assert int(idx.num_m_tiles.item()) == tiles
    te = torch.repeat_interleave(torch.arange(E, device=dev), padded // 128)
    assert torch.equal(idx.tile_expert[:tiles].long(), te)
    order = torch.argsort(ids.flatten(), stable=True)
    flat_e = ids.flatten()[order]
    rank = torch.arange(order.numel(), device=dev) - torch.cat([torch.zeros(1, dtype=torch.long, device=dev),
                                                                 cnt.cumsum(0)])[flat_e]
    expect_pos = torch.empty_like(order)
    expect_pos[order] = off[flat_e] + rank
    assert torch.equal(idx.pos.flatten().long(), expect_pos)
    src = torch.full((idx.rows,), -1, dtype=torch.long, device=dev)
    src[expect_pos] = torch.arange(order.numel(), device=dev)
    assert torch.equal(idx.row_src.long(), src)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case,H,N", [("mixed", 256, 384), ("mixed", 200, 136), ("one_expert", 128, 256),
                                      ("e128", 128, 128)])
def test_grouped_gemm_fwd_dgrad_wgrad(dtype, case, H, N):
    """Forward (K-major B), dgrad (MN-major B) and wgrad against an fp32 per-expert reference; N and K off the tile."""
    from torchacc_b200.ops.moe import grouped_gemm, grouped_wgrad
    dev = _dev()
    counts = COUNT_CASES[case]
    E = len(counts)
    ids = _ids_with_counts(counts, 1, dev)
    idx = _index(ids, E)
    T = ids.shape[0]
    torch.manual_seed(0)
    x = torch.randn(T, H, device=dev, dtype=dtype)
    w = (torch.randn(E, N, H, device=dev) / math.sqrt(H)).to(dtype)
    xp = _sorted_rows(idx, x)
    y = grouped_gemm(xp, w, idx)
    pos = idx.pos.long().flatten()
    ref = torch.einsum("th,tnh->tn", x.float(), w.float()[ids.flatten()])
    _close(y[pos], ref, 1e-2, 2e-2, "forward")
    # dgrad: dx = dy W_e
    dy = torch.randn(T, N, device=dev, dtype=dtype)
    dyp = _sorted_rows(idx, dy)
    dx = grouped_gemm(dyp, w, idx, b_mn_major=True)
    refdx = torch.einsum("tn,tnh->th", dy.float(), w.float()[ids.flatten()])
    _close(dx[pos], refdx, 1e-2, 2e-2 * math.sqrt(N / 64), "dgrad")
    # wgrad: dW_e = dy_e^T x_e, fp32 and 16-bit outputs, then accumulate into a view
    refdw = torch.zeros(E, N, H, device=dev)
    refdw.index_add_(0, ids.flatten(), torch.einsum("tn,th->tnh", dy.float(), x.float()))
    dw32 = grouped_wgrad(dyp, xp, idx, torch.full((E, N, H), float("nan"), device=dev))
    scale = max(1.0, math.sqrt(max(counts) / 64))
    _close(dw32, refdw, 1e-2, 2e-2 * scale, "wgrad fp32")
    dw16 = grouped_wgrad(dyp, xp, idx, torch.full((E, N, H), float("nan"), device=dev, dtype=dtype))
    _close(dw16, refdw, 2e-2, 2e-2 * scale, "wgrad 16-bit")
    flat = torch.randn(E * N * H + 8, device=dev)
    view = flat[8:].view(E, N, H)
    before = view.clone()
    grouped_wgrad(dyp, xp, idx, view, accumulate=True)
    _close(view, before + refdw, 1e-2, 2e-2 * scale, "wgrad accumulate")
    empty = [e for e, c in enumerate(counts) if c == 0]
    if empty:
        assert torch.equal(view[empty], before[empty]), "an empty expert changed under accumulate"
        assert bool((dw32[empty] == 0).all()), "an empty expert was not zeroed"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", ["mixed", "e128"])
def test_grouped_swiglu(dtype, case):
    from torchacc_b200.ops.moe import grouped_swiglu
    dev = _dev()
    counts = COUNT_CASES[case]
    E, H, Fd = len(counts), 192, 256
    ids = _ids_with_counts(counts, 1, dev)
    idx = _index(ids, E)
    T = ids.shape[0]
    torch.manual_seed(1)
    x = torch.randn(T, H, device=dev, dtype=dtype)
    w = (torch.randn(E, 2 * Fd, H, device=dev) / math.sqrt(H)).to(dtype)
    xp = _sorted_rows(idx, x)
    gu = torch.empty((idx.rows, 2 * Fd), device=dev, dtype=dtype)
    h = grouped_swiglu(xp, w, idx, gu)
    pos = idx.pos.long().flatten()
    rgu = torch.einsum("th,tnh->tn", x.float(), w.float()[ids.flatten()])
    _close(gu[pos], rgu, 1e-2, 2e-2, "pre-activation")
    _close(h[pos], F.silu(rgu[:, :Fd]) * rgu[:, Fd:], 2e-2, 2e-2, "h")


@pytest.mark.parametrize("E,k,norm", [(8, 2, True), (64, 8, False), (128, 8, True), (256, 4, True)])
def test_router_matches_softmax_topk(E, k, norm):
    from torchacc_b200.ops.moe import moe_router, moe_router_reference
    dev = _dev()
    torch.manual_seed(2)
    T = 300
    logits = (torch.randn(T, E, device=dev) + torch.arange(E, device=dev) * 1e-3).requires_grad_(True)
    w, ids = moe_router(logits, k, norm)
    lr = logits.detach().clone().requires_grad_(True)
    wr, idr = moe_router_reference(lr, k, norm)
    assert torch.equal(ids, idr)
    _close(w, wr, 1e-5, 1e-6, "weights")
    g = torch.randn_like(w)
    (w * g).sum().backward()
    (wr * g).sum().backward()
    _close(logits.grad, lr.grad, 1e-4, 1e-6, "dlogits")


def _hf_experts_loop(x, ids, w, wgu, wd):
    """HF's eager experts loop (MixtralExperts.forward) in fp32."""
    out = torch.zeros_like(x)
    E = wgu.shape[0]
    mask = F.one_hot(ids, num_classes=E).permute(2, 1, 0)
    for e in range(E):
        slot, tok = torch.where(mask[e])
        if tok.numel() == 0:
            continue
        gate, up = F.linear(x[tok], wgu[e]).chunk(2, dim=-1)
        y = F.linear(F.silu(gate) * up, wd[e]) * w[tok, slot, None]
        out = out.index_add(0, tok, y)
    return out


def _experts_case(dev, dtype, T=512, H=256, Fd=384, E=8, k=2, seed=3):
    torch.manual_seed(seed)
    x = torch.randn(T, H, device=dev, dtype=dtype)
    logits = torch.randn(T, E, device=dev)
    w, ids = torch.topk(torch.softmax(logits, -1), k, -1)
    w = w / w.sum(-1, keepdim=True)
    wgu = (torch.randn(E, 2 * Fd, H, device=dev) / math.sqrt(H)).to(dtype)
    wd = (torch.randn(E, H, Fd, device=dev) / math.sqrt(Fd)).to(dtype)
    return x, ids, w, wgu, wd


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("residual", [False, True])
def test_moe_experts_matches_hf_loop(dtype, residual):
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops.moe import moe_experts
    dev = _dev()
    x, ids, w, wgu, wd = _experts_case(dev, dtype)
    res = torch.randn_like(x) if residual else None
    leaves = [t.clone().requires_grad_(True) for t in (x, w, wgu, wd)]
    ref_leaves = [t.detach().float().clone().requires_grad_(True) for t in (x, w, wgu, wd)]
    n0 = nat.LAUNCHES
    out = moe_experts(leaves[0], ids, leaves[1], leaves[2], leaves[3], residual=res)
    ref = _hf_experts_loop(ref_leaves[0], ids, ref_leaves[1], ref_leaves[2], ref_leaves[3])
    if residual:
        ref = ref + res.float()
    _close(out, ref, 2e-2, 2e-2, "out")
    g = torch.randn_like(out)
    out.backward(g)
    ref.backward(g.float())
    assert nat.LAUNCHES - n0 >= 10, "native MoE kernels did not run"
    for name, a, b in zip(("dx", "dweights", "dW_gate_up", "dW_down"), leaves, ref_leaves):
        scale = b.grad.abs().max().item()
        # the 16-bit intermediates (pre-activation, dh, dgu) bound the error relative to the gradient's scale
        _close(a.grad, b.grad, 3e-2, 1e-2 * scale + 1e-2, name)


def test_moe_no_host_sync():
    from torchacc_b200.ops.moe import moe_experts, moe_router
    dev = _dev()
    x, ids, w, wgu, wd = _experts_case(dev, torch.bfloat16)
    logits = torch.randn(x.shape[0], 8, device=dev, dtype=torch.bfloat16, requires_grad=True)
    leaves = [t.clone().requires_grad_(True) for t in (x, wgu, wd)]
    moe_router(logits, 2, True)   # warm-up (library load, device query)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        wr, idr = moe_router(logits, 2, True)
        out = moe_experts(leaves[0], idr, wr, leaves[1], leaves[2])
        out.float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert logits.grad is not None and leaves[1].grad is not None


def test_moe_bitwise_deterministic():
    from torchacc_b200.ops.moe import moe_experts, moe_router
    dev = _dev()
    x, ids, w, wgu, wd = _experts_case(dev, torch.bfloat16, T=1024, E=16, k=4)
    logits = torch.randn(x.shape[0], 16, device=dev, dtype=torch.bfloat16)
    g = torch.randn_like(x)
    results = []
    for _ in range(3):
        leaves = [t.clone().requires_grad_(True) for t in (x, logits, wgu, wd)]
        wr, idr = moe_router(leaves[1], 4, True)
        out = moe_experts(leaves[0], idr, wr, leaves[2], leaves[3])
        out.backward(g)
        results.append([out.detach()] + [t.grad for t in leaves])
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a, b)


def _tiny_moe(dev, **kw):
    from torchacc_b200.models import build_llama
    with torch.device(dev):
        return build_llama("tiny-moe", dtype=torch.bfloat16, **kw)


def test_native_tiny_moe_matches_hf_mixtral():
    transformers = pytest.importorskip("transformers")
    dev = _dev()
    torch.manual_seed(0)
    model = _tiny_moe(dev)
    c = model.config
    hcfg = transformers.MixtralConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size,
                                      intermediate_size=c.moe_intermediate_size, num_hidden_layers=c.num_hidden_layers,
                                      num_attention_heads=c.num_attention_heads,
                                      num_key_value_heads=c.num_key_value_heads, head_dim=c.head_dim,
                                      num_local_experts=c.num_experts, num_experts_per_tok=c.num_experts_per_tok,
                                      rms_norm_eps=c.rms_norm_eps, rope_theta=c.rope_theta,
                                      max_position_embeddings=c.max_position_embeddings, tie_word_embeddings=False,
                                      router_aux_loss_coef=0.0)
    hf = transformers.MixtralForCausalLM(hcfg).to(dev, torch.bfloat16)
    model.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, c.vocab_size, (2, 128), device=dev)
    with torch.no_grad():
        ours = float(model(input_ids=ids, labels=ids)["loss"])
        ref = float(hf(input_ids=ids, labels=ids).loss)
    assert abs(ours - ref) < 2e-2 * max(1.0, abs(ref)), (ours, ref)
    back = model.to_hf_state_dict()
    for kname, v in hf.state_dict().items():
        assert torch.equal(back[kname].to(v.device), v), kname


def _train_tiny_moe(steps=4, seed=0):
    import torchacc_b200 as ta
    dev = _dev()
    torch.manual_seed(seed)
    model = _tiny_moe(dev)
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.compute.deterministic = True
    cfg.memory.gc = True
    cfg.memory.gc_cls = {"LlamaDecoderLayer"}
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=3e-3)
    g = torch.Generator(device=dev).manual_seed(seed)
    ids = torch.randint(0, model.config.vocab_size if hasattr(model, "config") else 512, (2, 256), device=dev,
                        generator=g)
    losses = []
    for _ in range(steps):
        out = model(input_ids=ids, labels=ids)
        out["loss"].backward()
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        losses.append(out["loss"].detach().clone())
    params = [p.detach().clone() for p in model.parameters()]
    return losses, params


def test_native_tiny_moe_training_bitwise_and_decreasing():
    from torchacc_b200 import _native as nat
    n0 = nat.LAUNCHES
    l1, p1 = _train_tiny_moe()
    assert nat.LAUNCHES > n0
    l2, p2 = _train_tiny_moe()
    for a, b in zip(l1, l2):
        assert torch.equal(a, b)
    for a, b in zip(p1, p2):
        assert torch.equal(a, b)
    assert float(l1[-1]) < float(l1[0]), [float(v) for v in l1]


@pytest.fixture
def restore_moe_classes():
    """Class-level patches are process-global: put every patched HF forward back after the test."""
    import importlib
    saved = []
    for mod, names in (("transformers.models.mixtral.modeling_mixtral", ("MixtralExperts", "MixtralRMSNorm",
                                                                          "MixtralForCausalLM")),
                       ("transformers.models.qwen3_moe.modeling_qwen3_moe", ("Qwen3MoeExperts", "Qwen3MoeRMSNorm",
                                                                              "Qwen3MoeMLP", "Qwen3MoeForCausalLM"))):
        m = importlib.import_module(mod)
        for n in names:
            cls = getattr(m, n)
            saved.append((cls, dict(cls.__dict__)))
    yield
    for cls, d in saved:
        for attr in ("forward", "_tb_orig_forward", "_tb_lce_patched"):
            if attr in d:
                setattr(cls, attr, d[attr])
            elif attr in cls.__dict__:
                delattr(cls, attr)


def _fix_routing(model, table):
    """Forward hooks on every router: keep HF's probabilities, but route each token to the experts in `table[layer]`
    (weights = its renormalised probabilities there), so two differently rounded runs take the same routing."""
    hooks = []
    for i, layer in enumerate(model.model.layers):
        def hook(mod, inp, out, _ids=table[i]):
            probs = out[0]
            w = probs.gather(-1, _ids)
            return probs, w / w.sum(-1, keepdim=True), _ids
        hooks.append(layer.mlp.gate.register_forward_hook(hook))
    return hooks


@pytest.mark.parametrize("family", ["mixtral", "qwen3_moe"])
def test_hf_moe_patch_preserves_loss_and_grads(family, restore_moe_classes, monkeypatch):
    """Patched bf16 model against an unpatched fp32 copy with the same (fixed) routing, aux loss on."""
    import copy
    transformers = pytest.importorskip("transformers")
    import torchacc_b200 as ta
    from torchacc_b200.ops import moe as moe_mod
    dev = _dev()
    torch.manual_seed(0)
    common = dict(vocab_size=256, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                  head_dim=64, max_position_embeddings=256, num_experts_per_tok=2, tie_word_embeddings=False,
                  output_router_logits=True, router_aux_loss_coef=0.02)
    if family == "mixtral":
        cfg = transformers.MixtralConfig(intermediate_size=256, num_local_experts=8, **common)
        model = transformers.MixtralForCausalLM(cfg)
        patch, E = ta.ops.apply_liger_kernel_to_mixtral, 8
    else:
        cfg = transformers.Qwen3MoeConfig(intermediate_size=512, moe_intermediate_size=256, num_experts=16,
                                          norm_topk_prob=True, decoder_sparse_step=1, **common)
        model = transformers.Qwen3MoeForCausalLM(cfg)
        patch, E = ta.ops.apply_liger_kernel_to_qwen3_moe, 16
    B, S, k = 2, 128, 2
    g = torch.Generator(device=dev).manual_seed(3)
    ids = torch.randint(0, 256, (B, S), device=dev, generator=g)
    table = [torch.rand(B * S, E, device=dev, generator=g).argsort(-1)[:, :k] for _ in range(cfg.num_hidden_layers)]
    ref_model = copy.deepcopy(model).to(dev)                      # fp32, unpatched
    _fix_routing(ref_model, table)
    ref = ref_model(input_ids=ids, labels=ids)
    ref.loss.backward()
    ref_grads = {n: p.grad.clone() for n, p in ref_model.named_parameters()}

    model = model.to(dev, torch.bfloat16)
    _fix_routing(model, table)
    patch()
    calls = []
    orig_apply = moe_mod._MoEExpertsFn.apply
    monkeypatch.setattr(moe_mod._MoEExpertsFn, "apply", lambda *a: calls.append(1) or orig_apply(*a))
    out = model(input_ids=ids, labels=ids)
    out.loss.backward()
    assert len(calls) == cfg.num_hidden_layers, "the experts did not run on the native kernels"
    assert out.aux_loss is not None and out.router_logits is not None
    assert abs(float(out.aux_loss) - float(ref.aux_loss)) < 1e-2 * float(ref.aux_loss)
    assert abs(float(out.loss) - float(ref.loss)) < 1e-2, (float(out.loss), float(ref.loss))
    for n, p in model.named_parameters():
        r = ref_grads[n]
        rel = float((p.grad.float() - r).norm() / r.norm())
        assert rel < 3e-2, (n, rel)


def test_moe_experts_sentinel_ids_residual_only_and_misaligned_inputs():
    """Ids outside [0, E) (HF's "no expert" sentinel E) add nothing and get zero d(weights); a residual-only backward;
    x / residual / d(out) on storage that is not 16-byte aligned."""
    from torchacc_b200.ops.moe import moe_experts, moe_experts_reference
    dev = _dev()
    x, ids, w, wgu, wd = _experts_case(dev, torch.bfloat16, T=256)
    E = wgu.shape[0]
    ids = ids.clone()
    ids[::7, 1] = E
    buf = torch.randn(x.numel() + 1, device=dev, dtype=x.dtype)
    xm = buf[1:].view_as(x)                                       # 2-byte offset
    xm.copy_(x)
    res_buf = torch.randn(x.numel() + 1, device=dev, dtype=x.dtype)
    res = res_buf[1:].view_as(x)
    wl = w.clone().requires_grad_(True)
    out = moe_experts(xm, ids, wl, wgu, wd, residual=res)
    ref = moe_experts_reference(x, ids, w, wgu, wd, residual=res)
    _close(out, ref, 2e-2, 2e-2, "out")
    gbuf = torch.randn(x.numel() + 1, device=dev, dtype=x.dtype)
    out.backward(gbuf[1:].view_as(x))
    assert bool((wl.grad[::7, 1] == 0).all()), "a sentinel id got a non-zero weight gradient"
    assert bool(torch.isfinite(wl.grad).all())
    r = torch.randn_like(x, requires_grad=True)
    out2 = moe_experts(x, ids, w, wgu, wd, residual=r)
    out2.backward(torch.ones_like(out2))
    assert torch.equal(r.grad, torch.ones_like(x))


def test_moe_mlp_with_aux_loss_has_no_host_sync():
    from torchacc_b200.ops.moe import MoEMLP, load_balancing_loss
    dev = _dev()
    torch.manual_seed(0)
    with torch.device(dev):
        mlp = MoEMLP(256, 256, 8, 2, dtype=torch.bfloat16)
    for p in mlp.parameters():
        torch.nn.init.normal_(p, 0, 0.05)
    x = torch.randn(512, 256, device=dev, dtype=torch.bfloat16, requires_grad=True)
    mlp(x)                                                        # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = mlp(x, residual=x)
        aux = load_balancing_loss([mlp.last_router_logits], [mlp.last_counts], 8)
        (out.float().sum() + aux).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    ref = load_balancing_loss([mlp.last_router_logits],
                              [F.one_hot(torch.topk(mlp.last_router_logits.float(), 2)[1].flatten(), 8).sum(0)], 8)
    assert abs(float(aux) - float(ref)) < 1e-5
    assert mlp.gate.weight.grad is not None
