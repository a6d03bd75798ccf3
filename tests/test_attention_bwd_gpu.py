"""Attention backward at head dim 64, where the main kernel uses 128-row query tiles and reduces dQ with TMA bulk
reduce-adds: ragged tails, short packed sequences, windows, GQA / MQA, ALiBi, dropout, fp16 and the phased blockwise
backward that accumulates several calls into one dQ accumulator.  Gradients are compared with the fp32 reference."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
D = 64


def _check(a, b, name, rtol=3e-2, atol=3e-2):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = int((err > tol).sum())
    assert bad == 0, f"{name}: {bad}/{a.numel()} off, max err {float(err.max()):.4g} (ref max {float(b.abs().max()):.3g})"


def _mk(seed, dtype=torch.bfloat16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lambda *shape: (torch.randn(*shape, device=DEV, generator=g) * 0.8).to(dtype)


CASES = [
    # dtype,         B, Sq,  Sk,  Hq, Hk, causal, window,    alibi, p
    (torch.bfloat16, 2, 200, 200, 4, 2, True, (-1, -1), False, 0.0),     # ragged 128-row tail
    (torch.bfloat16, 1, 130, 390, 4, 4, True, (-1, -1), False, 0.0),     # Sq != Sk, one row past a 128-row tile
    (torch.bfloat16, 2, 330, 330, 8, 2, False, (-1, -1), False, 0.0),    # GQA group of 4
    (torch.bfloat16, 1, 256, 256, 8, 1, True, (-1, -1), False, 0.0),     # GQA group of 8
    (torch.bfloat16, 1, 300, 300, 4, 1, False, (-1, -1), False, 0.0),    # MQA
    (torch.bfloat16, 1, 600, 600, 4, 2, True, (100, 0), False, 0.0),     # sliding window
    (torch.bfloat16, 1, 520, 520, 2, 2, False, (70, 30), False, 0.0),    # local, non-causal
    (torch.bfloat16, 2, 260, 260, 4, 2, True, (-1, -1), True, 0.0),      # ALiBi
    (torch.float16, 1, 200, 328, 4, 2, True, (64, 0), True, 0.0),        # fp16 + ALiBi + window
    (torch.float16, 2, 384, 384, 4, 4, False, (-1, -1), False, 0.0),     # fp16
    (torch.bfloat16, 1, 200, 328, 4, 2, False, (-1, -1), False, 0.1),    # dropout, ragged
    (torch.float16, 2, 256, 256, 8, 2, True, (-1, -1), False, 0.2),      # dropout, fp16
]


@pytest.mark.parametrize("dtype,B,Sq,Sk,Hq,Hk,causal,window,alibi,p", CASES)
def test_bwd_d64_matches_reference(dtype, B, Sq, Sk, Hq, Hk, causal, window, alibi, p):
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    mk = _mk(3, dtype)
    q, k, v, do = mk(B, Sq, Hq, D), mk(B, Sk, Hk, D), mk(B, Sk, Hk, D), mk(B, Sq, Hq, D)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    slopes = (torch.rand(B, Hq, device=DEV) * 0.3) if alibi else None
    torch.manual_seed(1234)
    out, _, keep = A.flash_attn_func(q, k, v, dropout_p=p, causal=causal, window_size=window, alibi_slopes=slopes,
                                     return_attn_probs=True)
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, _ = A.attention_reference(qf, kf, vf, None, causal, window, slopes, p, keep_mask=keep if p > 0 else None)
    ref.backward(do.float())
    tol = 3e-2 if dtype == torch.bfloat16 else 6e-3
    _check(out, ref, "out", tol, tol)
    _check(v.grad, vf.grad, "dv", tol, tol)
    _check(k.grad, kf.grad, "dk", tol, tol)
    _check(q.grad, qf.grad, "dq", tol, tol)
    A.set_attention_backend("auto")


@pytest.mark.parametrize("causal", [False, True])
def test_bwd_d64_packed_short_sequences(causal):
    """Packed sequences shorter than one 128-row query tile: a tile's rows past its sequence belong to the next one and
    must receive nothing but exact zeros from the dQ reduce-add."""
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    seqs = [37, 100, 5, 128, 90, 200]
    total, H, Hk = sum(seqs), 4, 2
    mk = _mk(9)
    q, k, v, do = mk(1, total, H, D), mk(1, total, Hk, D), mk(1, total, Hk, D), mk(1, total, H, D)
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    pos = torch.cat([torch.arange(n, device=DEV) for n in seqs])[None]
    out = A.flash_attn_varlen_position_ids_func(q, k, v, pos, causal=causal)
    out.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    refs, off = [], 0
    for n in seqs:
        r, _ = A.attention_reference(qf[:, off:off + n], kf[:, off:off + n], vf[:, off:off + n], None, causal)
        refs.append(r)
        off += n
    torch.cat(refs, 1).backward(do.float())
    _check(out, torch.cat(refs, 1), "out")
    _check(v.grad, vf.grad, "dv")
    _check(k.grad, kf.grad, "dk")
    _check(q.grad, qf.grad, "dq")
    A.set_attention_backend("auto")


def test_bwd_d64_blockwise_phases_into_one_dq_acc():
    """The blockwise backward that ring attention runs: phase 1 (delta, dq_acc = 0), phase 2 once per block (the two
    halves of the keys, then the two halves of the queries, 192 rows each, so tiles straddle the block edge), phase 4
    (cast) -- against one call with all phases."""
    from torchacc_b200.ops import attention as A
    from torchacc_b200.ops.context_parallel import ring as R
    A.set_attention_backend("native")
    B, S, Hq, Hk = 2, 384, 4, 2
    T, half, scale = B * S, S // 2, 1.0 / math.sqrt(D)
    mk = _mk(5)
    q, k, v, do = mk(B, S, Hq, D), mk(B, S, Hk, D), mk(B, S, Hk, D), mk(B, S, Hq, D)
    kv = torch.stack([k, v], 0)
    out, lse = R.ring_forward_native(q, [kv], [(0, "full")], scale)
    q3, o3, do3 = q.view(T, Hq, D), out.view(T, Hq, D), do.view(T, Hq, D)
    k3, v3 = kv.reshape(2, T, Hk, D)

    def run(calls):
        dq, dk, dv = torch.empty_like(q3), torch.zeros_like(k3), torch.zeros_like(v3)
        dq_acc = torch.empty((T, Hq, D), dtype=torch.float32, device=DEV)
        delta = torch.empty((Hq, T), dtype=torch.float32, device=DEV)
        for sk, view, phases, *sq in calls:
            R._blk_bwd(do3, q3, k3, v3, o3, lse, dq, dk, dv, dq_acc, delta, B, sq[0] if sq else S, sk, scale, False,
                       (-1, -1), view, phases)
        return dq, dk, dv

    none = (0, 0, 0, 0)
    full = run([(S, none, 7)])
    phased = run([(S, none, 1), (half, (0, 0, S, 0), 2), (half, (0, 0, S, half), 2), (S, none, 4)])
    for name, a, b in zip(("dq", "dk", "dv"), phased, full):
        _check(a, b, f"{name} phased vs one call", 1e-2, 1e-2)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref, _ = A.attention_reference(qf, kf, vf, scale, False)
    ref.backward(do.float())
    _check(phased[0].view(B, S, Hq, D), qf.grad, "dq")
    _check(phased[1].view(B, S, Hk, D), kf.grad, "dk")
    _check(phased[2].view(B, S, Hk, D), vf.grad, "dv")
    # query halves (ring's q_second_half view): the second call starts at q_off = 192, not a multiple of the 128-row
    # tile, and its last tile's rows past the half belong to the next sequence of the batch, which must get zeros only.
    # Each call writes dK / dV of all keys for its own queries, so only dQ accumulates across the two.
    dq_split = run([(S, none, 1), (S, (S, 0, 0, 0), 2, half), (S, (S, half, 0, 0), 2, half), (S, none, 4)])[0]
    _check(dq_split, full[0], "dq of query halves vs one call", 1e-2, 1e-2)
    _check(dq_split.view(B, S, Hq, D), qf.grad, "dq of query halves")
    A.set_attention_backend("auto")
