"""wgmma flash-attention kernels vs the explicit fp32 reference (causal / GQA / window / varlen / packed),
including the cases the reference's own suite skips (SURVEY section 4: causal, local, varlen-causal)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _rand(B, S, H, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(B, S, H, D, device=DEV, generator=g) * 0.8).bfloat16()


def _check(a, b, name, rtol=3e-2, atol=3e-2):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = int((err > tol).sum())
    assert bad == 0, f"{name}: {bad}/{a.numel()} off, max err {float(err.max()):.4g} (ref max {float(b.abs().max()):.3g})"


CASES = [
    # B, Sq, Sk, Hq, Hk, D, causal, window
    (2, 256, 256, 4, 4, 128, False, (-1, -1)),
    (2, 256, 256, 4, 4, 128, True, (-1, -1)),
    (1, 512, 512, 8, 2, 128, True, (-1, -1)),
    (2, 200, 200, 4, 2, 128, True, (-1, -1)),       # ragged tail
    (1, 130, 390, 4, 4, 128, True, (-1, -1)),       # Sq != Sk, bottom-right aligned causal
    (1, 384, 384, 4, 1, 64, True, (-1, -1)),        # head_dim 64, MQA
    (2, 320, 320, 4, 4, 64, False, (-1, -1)),
    (1, 640, 640, 4, 2, 128, True, (100, 0)),       # sliding window
    (1, 512, 512, 2, 2, 128, False, (64, 32)),      # local, non-causal
    (1, 1024, 1024, 8, 8, 128, True, (-1, -1)),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,D,causal,window", CASES)
def test_flash_attn_fwd_bwd(B, Sq, Sk, Hq, Hk, D, causal, window):
    from torchacc_b200.ops import attention as A
    from torchacc_b200 import _native as nat
    A.set_attention_backend("native")
    q, k, v = _rand(B, Sq, Hq, D, 1), _rand(B, Sk, Hk, D, 2), _rand(B, Sk, Hk, D, 3)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    n0 = nat.LAUNCHES
    out, lse, _ = A.flash_attn_func(q, k, v, causal=causal, window_size=window, return_attn_probs=True)
    assert nat.LAUNCHES > n0, "native attention kernel was not launched"
    do = _rand(B, Sq, Hq, D, 4)
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, lse_ref = A.attention_reference(qf, kf, vf, None, causal, window)
    ref.backward(do.float())
    _check(out, ref, "out")
    fin = torch.isfinite(lse_ref)
    _check(lse[fin], lse_ref[fin], "lse", 1e-2, 1e-2)
    _check(v.grad, vf.grad, "dv")
    _check(k.grad, kf.grad, "dk")
    _check(q.grad, qf.grad, "dq")
    A.set_attention_backend("auto")


def test_varlen_mask_and_position_ids():
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    B, S, H, Hk, D = 3, 256, 4, 2, 128
    q, k, v = _rand(B, S, H, D, 5), _rand(B, S, Hk, D, 6), _rand(B, S, Hk, D, 7)
    lens = torch.tensor([256, 100, 177], device=DEV)
    mask = (torch.arange(S, device=DEV)[None, :] < lens[:, None]).int()
    for causal in (False, True):
        out = A.flash_attn_varlen_func(q, k, v, mask, causal=causal)
        ref, _ = A.attention_reference_masked(q, k, v, mask.bool(), 1 / math.sqrt(D), causal, (-1, -1))
        _check(out, ref, f"varlen causal={causal}")
    # packed sequences by position ids (batch of 1)
    seqs = [100, 156, 128]
    total = sum(seqs)
    pos = torch.cat([torch.arange(n, device=DEV) for n in seqs])[None]
    q1, k1, v1 = _rand(1, total, H, D, 8), _rand(1, total, Hk, D, 9), _rand(1, total, Hk, D, 10)
    out = A.flash_attn_varlen_position_ids_func(q1, k1, v1, pos, causal=True)
    off = 0
    for n in seqs:
        ref, _ = A.attention_reference(q1[:, off:off + n], k1[:, off:off + n], v1[:, off:off + n], None, True)
        _check(out[:, off:off + n], ref, f"packed seq at {off}")
        off += n
    A.set_attention_backend("auto")


def test_qkvpacked_tokens_fwd_bwd():
    """The native-model fast path: fused QKV activation in, one dqkv tensor out."""
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    B, S, hq, hk, D = 2, 384, 8, 2, 128
    T = B * S
    g = torch.Generator(device=DEV).manual_seed(0)
    qkv = (torch.randn(T, (hq + 2 * hk) * D, device=DEV, generator=g) * 0.7).bfloat16().requires_grad_()
    out = A.flash_attn_qkvpacked_tokens(qkv, hq, hk, D, B, S, causal=True)
    do = (torch.randn(T, hq * D, device=DEV, generator=g)).bfloat16()
    out.backward(do)
    x = qkv.detach().float().requires_grad_()
    q = x[:, :hq * D].reshape(B, S, hq, D)
    k = x[:, hq * D:(hq + hk) * D].reshape(B, S, hk, D)
    v = x[:, (hq + hk) * D:].reshape(B, S, hk, D)
    ref, _ = A.attention_reference(q, k, v, None, True)
    ref.reshape(T, hq * D).backward(do.float())
    _check(out, ref.reshape(T, hq * D), "out")
    _check(qkv.grad, x.grad, "dqkv")
    A.set_attention_backend("auto")


# ---- reference parametrisation (tests/ops/test_flash_attn.py:41-181): dtype x mha/mqa/gqa x alibi x local x causal x
# head_dim {32, 96, 111 -> n/a (not a multiple of 8), 128} x seqlen pairs -- including the cases the reference skips
FEATURE_CASES = [
    # dtype,        B, Sq,  Sk,  Hq, Hk, D,   causal, window,    alibi
    (torch.float16, 2, 256, 256, 4, 4, 128, True, (-1, -1), False),
    (torch.float16, 1, 384, 384, 8, 2, 64, False, (-1, -1), False),
    (torch.float16, 1, 200, 328, 4, 1, 128, True, (64, 0), True),
    (torch.bfloat16, 2, 256, 256, 4, 4, 128, True, (-1, -1), True),       # ALiBi, causal
    (torch.bfloat16, 1, 130, 390, 4, 2, 128, False, (-1, -1), True),      # ALiBi, Sq != Sk, non-causal
    (torch.bfloat16, 1, 512, 512, 6, 6, 64, True, (128, 0), True),        # ALiBi + sliding window
    (torch.bfloat16, 2, 256, 256, 4, 2, 32, True, (-1, -1), False),       # head_dim 32 (zero-padded to 64)
    (torch.bfloat16, 1, 320, 320, 4, 4, 96, False, (-1, -1), False),      # head_dim 96 (padded to 128)
    (torch.float16, 1, 256, 256, 2, 2, 96, True, (-1, -1), True),         # fp16 + head_dim 96 + ALiBi
]


@pytest.mark.parametrize("dtype,B,Sq,Sk,Hq,Hk,D,causal,window,alibi", FEATURE_CASES)
def test_flash_attn_features(dtype, B, Sq, Sk, Hq, Hk, D, causal, window, alibi):
    from torchacc_b200.ops import attention as A
    from torchacc_b200 import _native as nat
    A.set_attention_backend("native")
    g = torch.Generator(device="cuda").manual_seed(7)
    mk = lambda *shape: (torch.randn(*shape, device="cuda", generator=g) * 0.8).to(dtype)
    q, k, v = mk(B, Sq, Hq, D), mk(B, Sk, Hk, D), mk(B, Sk, Hk, D)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    slopes = (torch.rand(B, Hq, device="cuda", generator=g) * 0.3) if alibi else None
    n0 = nat.LAUNCHES
    out, lse, _ = A.flash_attn_func(q, k, v, causal=causal, window_size=window, alibi_slopes=slopes,
                                    return_attn_probs=True)
    assert nat.LAUNCHES > n0, "native attention kernel was not launched"
    assert out.dtype == dtype and out.shape == q.shape
    do = mk(B, Sq, Hq, D)
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, lse_ref = A.attention_reference(qf, kf, vf, None, causal, window, slopes)
    ref.backward(do.float())
    tol = 2e-2 if dtype == torch.bfloat16 else 6e-3
    _check(out, ref, "out", tol, tol)
    fin = torch.isfinite(lse_ref)
    _check(lse[fin], lse_ref[fin], "lse", 1e-2, 1e-2)
    _check(v.grad, vf.grad, "dv", tol, tol)
    _check(k.grad, kf.grad, "dk", tol, tol)
    _check(q.grad, qf.grad, "dq", tol, tol)


@pytest.mark.parametrize("S", [4096, 8192])
def test_flash_attn_long_sequence(S):
    """the bench shape (B=2, H=32/8, D=128, causal) and twice its length: forward + backward vs the fp32 oracle on a
    head subset (the oracle materialises [H, S, S])"""
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    B, Hq, Hk, D = 1, 8, 2, 128
    g = torch.Generator(device="cuda").manual_seed(11)
    mk = lambda *shape: (torch.randn(*shape, device="cuda", generator=g) * 0.7).bfloat16()
    q, k, v = mk(B, S, Hq, D), mk(B, S, Hk, D), mk(B, S, Hk, D)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    out = A.flash_attn_func(q, k, v, causal=True)
    do = mk(B, S, Hq, D)
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, _ = A.attention_reference(qf, kf, vf, None, True, (-1, -1))
    ref.backward(do.float())
    _check(out, ref, "out")
    _check(q.grad, qf.grad, "dq", 3e-2, 3e-2)
    _check(k.grad, kf.grad, "dk", 3e-2, 3e-2)
    _check(v.grad, vf.grad, "dv", 3e-2, 3e-2)


# ---- blockwise (ring) kernels: every rank of a cp-way ring simulated on one GPU ---------------------------------------
def _shard(x, r, cp, zigzag):
    if zigzag:
        c = x.chunk(2 * cp, dim=1)
        return torch.cat([c[r], c[2 * cp - 1 - r]], 1).contiguous()
    return x.chunk(cp, dim=1)[r].contiguous()


def _unshard(parts, cp, zigzag):
    if not zigzag:
        return torch.cat(parts, 1)
    chunks = [None] * (2 * cp)
    for r, p in enumerate(parts):
        a, b = p.chunk(2, dim=1)
        chunks[r], chunks[2 * cp - 1 - r] = a, b
    return torch.cat(chunks, 1)


RING_CASES = [
    # cp, S_total, Hq, Hk, D, causal, zigzag, varlen
    (4, 2048, 4, 2, 128, True, True, False),
    (4, 1536, 4, 2, 128, True, True, False),       # half-chunk of 192 rows: tiles straddle the in-place half views
    (2, 512, 4, 4, 64, True, True, False),
    (4, 1024, 4, 2, 128, True, False, False),      # contiguous layout: rank r visits r + 1 blocks
    (4, 1024, 4, 2, 128, False, False, False),
    (4, 1024, 4, 2, 128, False, False, True),      # non-causal with per-sequence key lengths (packed cu_seqlens path)
]


@pytest.mark.parametrize("cp,S,Hq,Hk,D,causal,zigzag,varlen", RING_CASES)
def test_ring_blockwise_kernels_match_full_attention(cp, S, Hq, Hk, D, causal, zigzag, varlen):
    """ring_forward_native / ring_backward_native (in-kernel merge, in-place half-block views, phased backward with
    one shared dQ accumulator) for every rank of the ring vs one full-sequence fp32 attention."""
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import attention as A
    from torchacc_b200.ops.context_parallel import ring as R
    A.set_attention_backend("native")
    B = 2
    q, k, v, do = _rand(B, S, Hq, D, 1), _rand(B, S, Hk, D, 2), _rand(B, S, Hk, D, 3), _rand(B, S, Hq, D, 4)
    scale = 1.0 / math.sqrt(D)
    k_lens = torch.tensor([S, S * 5 // 8 + 37], device=DEV, dtype=torch.int32) if varlen else None
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    if varlen:
        mask = (torch.arange(S, device=DEV)[None] < k_lens[:, None])
        g = Hq // Hk
        s = torch.einsum("bqhd,bkhd->bhqk", qf, kf.repeat_interleave(g, 2)) * scale
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
        ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf.repeat_interleave(g, 2))
    else:
        ref, _ = A.attention_reference(qf, kf, vf, scale, causal, (-1, -1))
    ref.backward(do.float())
    assert R.native_blockwise_ok(q, k, v)
    zig = zigzag and causal
    blocks = [torch.stack([_shard(k, j, cp, zig), _shard(v, j, cp, zig)], 0) for j in range(cp)]
    outs, dqs, dkv_sum = [], [], None
    for r in range(cp):
        steps = R._plan(r, cp, causal, zig)
        q_r, do_r = _shard(q, r, cp, zig), _shard(do, r, cp, zig)
        n0 = nat.LAUNCHES
        out_r, lse_r = R.ring_forward_native(q_r, blocks, steps, scale, k_lens=k_lens)
        assert nat.LAUNCHES - n0 == len(steps), "one kernel launch per ring step"
        dq_r, dkv_r = R.ring_backward_native(do_r, q_r, out_r, lse_r, blocks, steps, scale, k_lens=k_lens)
        outs.append(out_r)
        dqs.append(dq_r)
        dkv_sum = dkv_r.float() if dkv_sum is None else dkv_sum + dkv_r.float()
    out = _unshard(outs, cp, zig)
    dq = _unshard(dqs, cp, zig)
    dk = _unshard([dkv_sum[j, 0] for j in range(cp)], cp, zig)
    dv = _unshard([dkv_sum[j, 1] for j in range(cp)], cp, zig)
    _check(out, ref, "out")
    _check(dq, qf.grad, "dq")
    _check(dk, kf.grad, "dk")
    _check(dv, vf.grad, "dv")


# ---- dropout: counter-based mask regenerated by the backward -----------------------------------------------------------
DROPOUT_CASES = [
    # B, Sq, Sk, Hq, Hk, D, causal, p
    (2, 256, 256, 4, 2, 128, True, 0.17),
    (1, 200, 328, 4, 4, 64, False, 0.1),          # ragged tiles, Sq != Sk
    (2, 384, 384, 8, 2, 128, True, 0.5),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,D,causal,p", DROPOUT_CASES)
def test_flash_attn_dropout_matches_reference_with_the_same_mask(B, Sq, Sk, Hq, Hk, D, causal, p):
    """Native attention dropout (reference flash_attn.py:313-355 keeps a Philox state; ours is a counter-based hash of
    (seed, head, q, k), csrc/attn/dropout.cuh): forward and backward agree with the fp32 reference that applies the
    SAME keep mask (rebuilt in PyTorch by dropout_keep_mask), and the mask drops about p of the entries."""
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    q, k, v, do = _rand(B, Sq, Hq, D, 1), _rand(B, Sk, Hk, D, 2), _rand(B, Sk, Hk, D, 3), _rand(B, Sq, Hq, D, 4)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    torch.manual_seed(1234)
    n0 = nat.LAUNCHES
    out, lse, keep = A.flash_attn_func(q, k, v, dropout_p=p, causal=causal, return_attn_probs=True)
    assert nat.LAUNCHES > n0, "native attention kernel was not launched"
    assert keep.shape == (B, Hq, Sq, Sk) and keep.dtype == torch.bool
    frac = float((~keep).float().mean())
    assert abs(frac - p) < 0.01, frac
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, lse_ref = A.attention_reference(qf, kf, vf, None, causal, (-1, -1), None, p, keep_mask=keep)
    ref.backward(do.float())
    _check(out, ref, "out")
    fin = torch.isfinite(lse_ref)
    _check(lse[fin], lse_ref[fin], "lse", 1e-2, 1e-2)          # the statistics are those of the undropped softmax
    _check(v.grad, vf.grad, "dv")
    _check(k.grad, kf.grad, "dk")
    _check(q.grad, qf.grad, "dq")
    # same seed -> same result; a different seed -> a different mask
    torch.manual_seed(1234)
    again = A.flash_attn_func(q.detach(), k.detach(), v.detach(), dropout_p=p, causal=causal)
    assert torch.equal(again, out.detach())
    other = A.flash_attn_func(q.detach(), k.detach(), v.detach(), dropout_p=p, causal=causal)
    assert not torch.equal(other, out.detach())
