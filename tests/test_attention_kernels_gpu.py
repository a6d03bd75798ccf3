"""The attention kernels (csrc/attn/flash_fwd.cu, flash_bwd.cu) against fp64 references computed from the exact 16-bit
inputs, with error bounds derived from the kernels' arithmetic, at peaked logits, mask edges and every launch variant.

The arithmetic contract the bounds rely on (and nothing more, so that a restructured kernel keeping it still passes):
  * scores S = Q K^T are accumulated in fp32 over D; the softmax runs in log2 units with ``ex2.approx.ftz``;
  * P is rounded once to the 16-bit type before P V (dropout: P * keep / (1 - p), rounded once); the row sum l is an
    fp32 sum of P (unrounded or rounded: both are covered), over key tiles in any order;
  * the backward recomputes P from the forward's LSE, delta = rowsum(dO o O) uses the rounded O, dS = P o (dP - delta)
    is rounded to 16 bits before dQ = scale dS K and dK = scale dS^T Q, and dQ / dK / dV are accumulated in fp32.
Rows that see no key follow FlashAttention-2: O = 0, LSE = -inf, dQ = 0.

Every bound is (1 ulp of the output dtype, the final rounding) + (1 + u) x a floor built from absolute-value products of
the reference (P|V|, P^T|dO|, |dS||K|, |dS|^T|Q|, sum |q||k|); the derivation of each term is written next to it in
``_reference``.  ``[ulp]`` lines print the largest fraction of each bound that was used."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
U32 = 2.0 ** -24          # fp32 unit roundoff
FTZ = 2.0 ** -126         # ex2.approx.ftz flushes results below the smallest fp32 normal to zero
KAPPA = 0.02              # second-order slack of the first-order bounds (asserted below: every relative error < 2^-6)


@pytest.fixture(autouse=True)
def _native_backend():
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    yield
    A.set_attention_backend("auto")


# ---------------------------------------------------------------------------------------------------------------------
# helpers (the conventions of test_ops_kernels_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
def ulp_dtype(ref64, dtype):
    """Spacing of ``dtype`` at |ref| (2^floor(log2 |ref|) * eps); below the smallest normal number, the subnormal
    spacing."""
    fi = torch.finfo(dtype)
    return torch.exp2(torch.floor(torch.log2(ref64.abs().clamp(min=fi.tiny)))) * fi.eps


def check(out, ref64, what, ulps=1.0, floor=None, dtype=None):
    """Every element within ``ulps`` ulps of the fp64 reference plus ``floor``.  NaN fails.  Prints the largest ulp
    error and the largest fraction of the bound used."""
    dtype = dtype or out.dtype
    err = (out.double() - ref64).abs()
    tol = ulps * ulp_dtype(ref64, dtype) + (0.0 if floor is None else floor)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} outside {ulps} ulp + floor; first at flat index "
                             f"{i}: out {out.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r} "
                             f"tol {tol.reshape(-1)[i].item():.3g}")
    used = float((err / tol).max()) if out.numel() else 0.0
    print(f"[ulp] {what}: {used:.3f} of the bound")
    return used


def _visible(q_len, k_len, causal, window, device=None):
    """bool [q_len, k_len]: key j visible to query row i (bottom-right aligned causal / window, FA2 semantics)."""
    device = device or DEV
    pos = torch.arange(q_len, device=device)[:, None] + (k_len - q_len)
    j = torch.arange(k_len, device=device)[None, :]
    wl, wr = window
    r = (0 if wr < 0 else min(wr, 0)) if causal else wr
    vis = torch.ones(q_len, k_len, dtype=torch.bool, device=device)
    if r >= 0:
        vis &= j <= pos + r
    if wl >= 0:
        vis &= j >= pos - wl
    return vis


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference and bounds
# ---------------------------------------------------------------------------------------------------------------------
def _reference(q3, k3, v3, do3, o3, lse_hat, cu_q, cu_k, scale, causal, window, alibi=None, keep=None, p_drop=0.0,
               blocks=1, backward=True):
    """Packed token-major inputs q3 / do3 [Tq, Hq, D], k3 / v3 [Tk, Hk, D] (the kernels' exact 16-bit values), the
    kernel's forward output o3 and LSE (lse_hat [Hq, Tq], or None: then its bound stands in for its error), python
    lists cu_q / cu_k.  alibi: fp32 [Hq] or [B, Hq]; keep(b) -> bool [Hq, q_len, k_len] (dropout keep mask).
    ``blocks`` > 1: the forward ran as that many blockwise (ring) calls merged in fp32.

    Returns fp64 o, lse, dq, dk, dv and their bounds bo, blse, bdq, bdk, bdv (floors before the final rounding)."""
    dtype = q3.dtype
    fi = torch.finfo(dtype)
    u = fi.eps / 2                         # unit roundoff of the 16-bit type
    h16 = fi.tiny * fi.eps / 2             # half the subnormal spacing: absolute rounding error near zero (fp16 P, dS)
    Tq, Hq, D = q3.shape
    Tk, Hk = k3.shape[:2]
    g = Hq // Hk
    f64 = dict(dtype=torch.float64, device=q3.device)
    R = {n: torch.zeros(Tq, Hq, D, **f64) for n in ("o", "bo", "dq", "bdq")}
    R.update({n: torch.zeros(Tk, Hk, D, **f64) for n in ("dk", "bdk", "dv", "bdv")})
    R["lse"] = torch.full((Hq, Tq), -math.inf, **f64)
    R["blse"] = torch.zeros(Hq, Tq, **f64)
    p32 = torch.tensor(p_drop, dtype=torch.float32)
    rp = float(1.0 / (1.0 - p32)) if p_drop > 0 else 1.0          # the kernels' fp32 1 / (1 - p)
    for b in range(len(cu_q) - 1):
        qs, qe, ks, ke = cu_q[b], cu_q[b + 1], cu_k[b], cu_k[b + 1]
        Sq, Sk = qe - qs, ke - ks
        if Sq == 0 or Sk == 0:
            continue                        # rows without keys keep O = 0, LSE = -inf, dQ = 0; keys without rows dK = 0
        vis = _visible(Sq, Sk, causal, window, q3.device)
        dist = (torch.arange(Sq, device=q3.device)[:, None] + (Sk - Sq)
                - torch.arange(Sk, device=q3.device)[None, :]).abs().double()
        n_t = -(-Sk // 128) + 1             # key tiles a row visits (+1: a restructured kernel may split differently)
        # fp32 row sum l (per lane at most a 256-key tile's quarter of sequential adds, then one add and one alpha
        # rescale, |ex2 error| <= 2^-22, per tile): relative error of l
        eps_l = (68 + 2 * n_t) * U32 + n_t * 4 * U32
        # fp32 tensor-core accumulation: each k16 step and each tile rescale adds at most 2^-22 of the running sum of
        # |terms|; plus the final 1 / l, merge and conversion multiplies
        eps_acc_o = (-(-Sk // 16) + n_t + 4) * 4 * U32
        eps_acc_k = (-(-Sk // 16) + -(-Sk // 64) + 8) * 4 * U32     # dQ: k16 steps + one reduce-add per 64-key partial
        eps_acc_q = (g * -(-Sq // 16) + 8) * 4 * U32                # dK / dV: k16 steps over every query of the group
        slopes = None
        if alibi is not None:
            slopes = (alibi[b] if alibi.dim() == 2 else alibi).double()
        hc = max(1, min(Hq, (1 << 26) // (Sq * Sk)))                # heads per chunk: <= 512 MB per fp64 [h, Sq, Sk]
        for h0 in range(0, Hq, hc):
            h1 = min(Hq, h0 + hc)
            kh = torch.arange(h0, h1, device=q3.device) // g
            qd = q3[qs:qe, h0:h1].double().transpose(0, 1)
            kd = k3[ks:ke].index_select(1, kh).double().transpose(0, 1)
            vd = v3[ks:ke].index_select(1, kh).double().transpose(0, 1)
            s = qd @ kd.transpose(1, 2) * scale
            A_ = qd.abs() @ kd.abs().transpose(1, 2)
            bias = torch.zeros_like(s) if slopes is None else -slopes[h0:h1].view(-1, 1, 1) * dist
            t = torch.where(vis, s + bias, -math.inf)
            lse = torch.logsumexp(t, -1)
            m = t.amax(-1)
            fin = torch.isfinite(lse)
            lse_f, m_f = torch.where(fin, lse, 0.0), torch.where(fin, m, 0.0)
            P = torch.where(vis & fin[..., None], torch.exp(t - lse_f[..., None]), 0.0)
            # Score error, natural-log units, per entry: the fp32 dot product over D (D u32 sum |q||k|, the worst case
            # of any summation order), times scale; the scale * log2e product, the ALiBi product and the fused
            # subtraction of the running max (forward) or the LSE (backward) each round once in fp32
            # (<= 2^-23 of |s scale| + 2 |bias| + |m| + |lse|); ex2.approx (relative error < 2^-22 < 2^-21 in ln).
            eps = torch.where(vis, scale * D * U32 * A_ + 4 * U32 * ((s.abs() + 2 * bias.abs()) + m_f.abs()[..., None]
                                                                       + lse_f.abs()[..., None]) + 2.0 ** -21, 0.0)
            del A_
            assert float((P * eps).amax()) < 2.0 ** -7 and u < 2.0 ** -7, "the first-order bounds need small errors"
            Kd = torch.ones_like(P) if keep is None else keep(b)[h0:h1].double() * rp
            Pd = P * Kd
            vabs = vd.abs()
            o = Pd @ vd
            PV = Pd @ vabs
            Pe = (P * eps).sum(-1, keepdim=True)
            if blocks > 1:
                # each ring block normalises with its own l and LSE: the block-weighted score error is at most the row
                # maximum, and it enters through O_blk / l_blk and through the merge weight exp(lse_blk - lse) (once
                # each, plus the merged LSE's error); every merge adds ~2^-21 (__expf, __logf, one division)
                Pe = 3 * eps.amax(-1, keepdim=True) + 2 * eps_l + blocks * 2.0 ** -19
            # O = sum_j P_j (1 + d_j)(1 + r_j) v_j / (l (1 + dbar + z)): d_j the score / exp2 error, r_j the rounding of
            # P to 16 bits (u, +2 u32 for the dropout factor), dbar = sum_j P_j d_j (+ u when l sums the rounded P),
            # z the error of the fp32 sum l.  First order: (P o eps)|V| + (u + Pe + u + eps_l) P|V|, plus the fp32
            # accumulation of P V, plus fp16's subnormal P (<= h16 absolute per key, relative to l >= 1 in max units)
            # ex2.approx.ftz flushes P (and alpha) below 2^-126 to zero: another 2^-126 absolute per key
            vsum = vis.double() @ vabs
            bo = (1 + KAPPA) * ((Pd * eps) @ vabs + (2 * u + 2 * U32 + Pe + eps_l + eps_acc_o) * PV) \
                + (FTZ + h16) * rp * vsum * torch.exp(m_f - lse_f)[..., None]
            # LSE = (m + log2 l) ln2: the P-weighted score error, the error of l, log2f / the two fp32 roundings of the
            # result (<= 2^-21 of |lse| + |log l| + 1)
            blse = (1 + KAPPA) * (Pe.squeeze(-1) + eps_l) + 2.0 ** -21 * ((lse_f - m_f).abs() + lse_f.abs() + 1)
            if blocks > 1:
                blse = blse + blocks * (2.0 ** -20 + 2.0 ** -22 * lse_f.abs())
            R["o"][qs:qe, h0:h1] = o.transpose(0, 1)
            R["bo"][qs:qe, h0:h1] = bo.transpose(0, 1)
            R["lse"][h0:h1, qs:qe] = lse
            R["blse"][h0:h1, qs:qe] = torch.where(fin, blse, 0.0)
            del s, bias, t, PV, vsum
            if not backward:
                continue
            dod = do3[qs:qe, h0:h1].double().transpose(0, 1)
            oh = o3[qs:qe, h0:h1].double().transpose(0, 1)
            dabs = dod.abs()
            dP = (dod @ vd.transpose(1, 2)) * Kd
            # fp32 dP over D (D u32 sum |dO||V|), times the fp32 dropout factor
            edP = Kd * D * U32 * (dabs @ vabs.transpose(1, 2)) + 2 * U32 * dP.abs()
            delta = (dod * o).sum(-1, keepdim=True)                  # = rowsum(P o dP), exactly
            # the kernels' delta is the fp32 dot product of dO with the rounded O: its error is measured, not bounded
            ddelta = (dabs * (oh - o).abs()).sum(-1, keepdim=True) + D * U32 * (dabs * oh.abs()).sum(-1, keepdim=True)
            if lse_hat is None:
                dlse = blse[..., None]
            else:
                lh = lse_hat[h0:h1, qs:qe].double()
                dlse = torch.where(fin, (lh - lse_f).abs(), 0.0)[..., None]
            theta = torch.where(vis, eps + dlse, 0.0)                # relative error of the backward's recomputed P
            dS = P * (dP - delta)
            # dS = P (dP - delta) scale: P off by theta, dP by edP, delta by ddelta; three fp32 roundings; then the
            # rounding to 16 bits (u relative, h16 absolute near zero)
            # (the recomputed P also flushes to zero below 2^-126)
            bpre = (1 + KAPPA) * (P * (theta * (dP - delta).abs() + edP + ddelta)
                                  + FTZ * vis * ((dP - delta).abs() + edP + ddelta)) + 4 * U32 * dS.abs()
            bdS = scale * ((1 + u) * bpre + u * dS.abs()) + h16 * vis.double()
            del edP, bpre
            dSa = scale * dS.abs()
            R["dq"][qs:qe, h0:h1] = (scale * dS @ kd).transpose(0, 1)
            R["bdq"][qs:qe, h0:h1] = (bdS @ kd.abs() + eps_acc_k * (dSa @ kd.abs())).transpose(0, 1)
            dk = scale * dS.transpose(1, 2) @ qd
            bdk = bdS.transpose(1, 2) @ qd.abs() + (eps_acc_q + (u if blocks > 1 else 0.0)) * (
                dSa.transpose(1, 2) @ qd.abs())
            dv = Pd.transpose(1, 2) @ dod
            # dV: P^T dO with P off by theta, rounded to 16 bits (+ the dropout factor), fp32 accumulation; ring: each
            # rank's dK / dV contribution is rounded to 16 bits before the ranks are summed (one more u)
            bdv = ((1 + KAPPA) * Pd * (theta + u + 2 * U32) + (FTZ + h16) * rp * vis.double()).transpose(1, 2) @ dabs \
                + (eps_acc_q + (u if blocks > 1 else 0.0)) * (Pd.transpose(1, 2) @ dabs)
            R["dk"][ks:ke].index_add_(1, kh, dk.transpose(0, 1))
            R["bdk"][ks:ke].index_add_(1, kh, bdk.transpose(0, 1))
            R["dv"][ks:ke].index_add_(1, kh, dv.transpose(0, 1))
            R["bdv"][ks:ke].index_add_(1, kh, bdv.transpose(0, 1))
    return R


def _check_fwd(tag, R, o3, lse_hat=None):
    dtype = o3.dtype
    u = torch.finfo(dtype).eps / 2
    check(o3, R["o"], f"{tag} O", floor=(1 + u) * R["bo"])
    if lse_hat is not None:
        none = ~torch.isfinite(R["lse"])
        assert bool((lse_hat[none] == -math.inf).all()), f"{tag}: rows without keys must have LSE = -inf"
        fin = ~none
        check(lse_hat[fin], R["lse"][fin], f"{tag} LSE", ulps=0, floor=R["blse"][fin], dtype=torch.float32)


def _check_bwd(tag, R, dq, dk, dv, ulps=1.0):
    u = torch.finfo(dq.dtype).eps / 2
    check(dq, R["dq"], f"{tag} dQ", ulps, floor=(1 + u) * R["bdq"], dtype=dq.dtype)
    check(dk, R["dk"], f"{tag} dK", ulps, floor=(1 + u) * R["bdk"], dtype=dq.dtype)
    check(dv, R["dv"], f"{tag} dV", ulps, floor=(1 + u) * R["bdv"], dtype=dq.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# input regimes
# ---------------------------------------------------------------------------------------------------------------------
def _row_bounds(cu_q, cu_k, causal, window, device=None):
    """Per packed query row: first / last visible key as packed key indices (lo > hi: none)."""
    device = device or DEV
    lo, hi = [], []
    for b in range(len(cu_q) - 1):
        Sq, Sk = cu_q[b + 1] - cu_q[b], cu_k[b + 1] - cu_k[b]
        if Sq == 0:
            continue
        if Sk == 0:
            lo.append(torch.ones(Sq, dtype=torch.long, device=device))
            hi.append(torch.zeros(Sq, dtype=torch.long, device=device))
            continue
        vis = _visible(Sq, Sk, causal, window, device)
        j = torch.arange(Sk, device=device)
        lo.append(cu_k[b] + torch.where(vis, j, Sk).amin(1))
        hi.append(cu_k[b] + torch.where(vis, j, -1).amax(1))
    return torch.cat(lo), torch.cat(hi)


def _make(regime, cu_q, cu_k, Hq, Hk, D, dtype, causal, window, scale, seed):
    """q3 [Tq, Hq, D], k3 / v3 [Tk, Hk, D], do3 [Tq, Hq, D] in ``dtype``.

    flat:   randn * 0.8 (scaled logits of standard deviation ~0.6 at D = 128: nearly uniform softmax).
    peaked: q, k ~ 2 randn (logits of standard deviation ~4), plus, per row, a boost of 5..40 (every 8th row: 100) on
            its first visible key (even rows) or its last (odd rows), so the row maximum arrives in the first tile (the
            later tiles' P flush to zero) or in the last one (alpha from ~1 down to flushed-to-zero).
    probe:  each row's logits peak (by ~5 above every other key) at the first invisible key on its left (rows of even
            row + head) or right (odd): positions are encoded as cos / sin of 2 pi 2^m t / L over 2 log2 L head-dim
            components (t: packed key index), so a mask that leaks the neighbouring key moves O by O(1).
    zero_q: q = 0 -- uniform attention over the visible keys."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    Tq, Tk = cu_q[-1], cu_k[-1]
    rn = lambda *s: torch.randn(*s, device=DEV, generator=gen, dtype=torch.float64)
    v, do = rn(Tk, Hk, D), rn(Tq, Hq, D)
    if regime == "flat":
        q, k, v, do = 0.8 * rn(Tq, Hq, D), 0.8 * rn(Tk, Hk, D), 0.8 * v, 0.8 * do
    elif regime == "zero_q":
        q, k = torch.zeros(Tq, Hq, D, dtype=torch.float64, device=DEV), rn(Tk, Hk, D)
    elif regime == "peaked":
        q, k = 2 * rn(Tq, Hq, D), 2 * rn(Tk, Hk, D)
        k = k.to(dtype).double()
        lo, hi = _row_bounds(cu_q, cu_k, causal, window)
        rows = torch.arange(Tq, device=DEV)
        tgt = torch.where(rows % 2 == 0, lo, hi).clamp(0, max(Tk - 1, 0))
        gamma = 5 + 35 * torch.rand(Tq, device=DEV, generator=gen, dtype=torch.float64)
        gamma[::8] = 100.0
        g = Hq // Hk
        kt = k[tgt].repeat_interleave(g, 1)                         # [Tq, Hq, D]: the target key of each row
        q = q + (gamma / scale)[:, None, None] * kt / kt.square().sum(-1, keepdim=True)
    elif regime == "probe":
        L = 1 << max(4, math.ceil(math.log2(Tk + 2)) + 1)
        n = int(math.log2(L))
        assert 2 * n <= D
        theta = 2 * math.pi * (2.0 ** torch.arange(n, device=DEV, dtype=torch.float64)) / L
        kpos = torch.arange(Tk, device=DEV, dtype=torch.float64)[:, None] * theta
        k = 0.3 * rn(Tk, Hk, D)
        k[:, :, :2 * n] = torch.cat([kpos.cos(), kpos.sin()], -1)[:, None, :]
        lo, hi = _row_bounds(cu_q, cu_k, causal, window)
        rows = torch.arange(Tq, device=DEV)[:, None]
        heads = torch.arange(Hq, device=DEV)[None, :]
        tgt = torch.where((rows + heads) % 2 == 0, lo[:, None] - 1, hi[:, None] + 1).double()   # [Tq, Hq]
        qpos = tgt[..., None] * theta
        q = 0.3 * rn(Tq, Hq, D) / math.sqrt(D)
        q[:, :, :2 * n] = (2.0 / scale) * torch.cat([qpos.cos(), qpos.sin()], -1)
    else:
        raise ValueError(regime)
    return q.to(dtype), k.to(dtype), v.to(dtype), do.to(dtype)


# ---------------------------------------------------------------------------------------------------------------------
# runners
# ---------------------------------------------------------------------------------------------------------------------
def _uniform(cu):
    return len(cu) > 1 and cu[1] > 0 and all(b - a == cu[1] for a, b in zip(cu, cu[1:]))


def _run_varlen(q3, k3, v3, do3, cu_q, cu_k, scale, causal, window, alibi=None, p=0.0, det=False):
    """Forward + backward through flash_attn_func (fixed-length batches: the kernels' q_bs / k_bs addressing) or
    flash_attn_varlen_cu (cu_seqlens).  Returns (o, lse [Hq, Tq], dq, dk, dv, keep(b) or None)."""
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import attention as A
    leaves = [t.detach().clone().requires_grad_() for t in (q3, k3, v3)]
    torch.manual_seed(4321)
    seed = A.new_dropout_seed()
    torch.manual_seed(4321)
    n0 = nat.LAUNCHES
    if _uniform(cu_q) and _uniform(cu_k):
        B, Sq, Sk = len(cu_q) - 1, cu_q[1], cu_k[1]
        Hq, D = q3.shape[1:]
        q4, k4, v4 = leaves[0].view(B, Sq, Hq, D), leaves[1].view(B, Sk, -1, D), leaves[2].view(B, Sk, -1, D)
        o, lse, dmask = A.flash_attn_func(q4, k4, v4, dropout_p=p, softmax_scale=scale, causal=causal,
                                          window_size=window, alibi_slopes=alibi, deterministic=det,
                                          return_attn_probs=True)
        assert nat.LAUNCHES > n0, "native attention kernel was not launched"
        o.backward(do3.view(B, Sq, Hq, D))
        keep = (lambda b: dmask[b]) if p > 0 else None
        return (o.detach().reshape(B * Sq, Hq, D), lse.permute(1, 0, 2).reshape(Hq, B * Sq), leaves[0].grad,
                leaves[1].grad, leaves[2].grad, keep)
    cq = torch.tensor(cu_q, dtype=torch.int32, device=DEV)
    ck = torch.tensor(cu_k, dtype=torch.int32, device=DEV)
    o, lse = A.flash_attn_varlen_cu(*leaves, cq, ck, scale, causal, window, return_lse=True, dropout_p=p,
                                    alibi_slopes=alibi, deterministic=det)
    assert nat.LAUNCHES > n0, "native attention kernel was not launched"
    o.backward(do3)
    keep = None
    if p > 0:
        Hq = q3.shape[1]
        Bn, mq = len(cu_q) - 1, max(b - a for a, b in zip(cu_q, cu_q[1:]))
        mk = max(b - a for a, b in zip(cu_k, cu_k[1:]))
        full = A.dropout_keep_mask(seed, p, Bn, Hq, mq, mk, DEV)
        keep = lambda b: full[b, :, :cu_q[b + 1] - cu_q[b], :cu_k[b + 1] - cu_k[b]]
    return o.detach(), lse, leaves[0].grad, leaves[1].grad, leaves[2].grad, keep


def _case(tag, cu_q, cu_k, Hq, Hk, D, dtype, causal, window, regime, scale=None, alibi=None, p=0.0, dets=(False,),
          seed=0):
    """Run the kernels (default and / or deterministic backward) on one packed problem and check everything against the
    fp64 reference.  With both backward paths, dK and dV must be bitwise equal between them."""
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    q3, k3, v3, do3 = _make(regime, cu_q, cu_k, Hq, Hk, D, dtype, causal, window, scale, seed)
    runs = {det: _run_varlen(q3, k3, v3, do3, cu_q, cu_k, scale, causal, window, alibi, p, det) for det in dets}
    o, lse, _, _, _, keep = runs[dets[0]]
    R = _reference(q3, k3, v3, do3, o, lse, cu_q, cu_k, scale, causal, window, alibi, keep, p)
    _check_fwd(tag, R, o, lse)
    for det, (o2, lse2, dq, dk, dv, _) in runs.items():
        assert torch.equal(o2, o) and torch.equal(lse2, lse)
        _check_bwd(f"{tag} {'det' if det else 'default'}", R, dq, dk, dv)
    if len(runs) == 2:
        (_, _, _, dk0, dv0, _), (_, _, _, dk1, dv1, _) = runs[False], runs[True]
        assert torch.equal(dk0, dk1) and torch.equal(dv0, dv1), "deterministic dK / dV differ from the default path"
    return R, runs


def _fixed(B, Sq, Sk):
    return [b * Sq for b in range(B + 1)], [b * Sk for b in range(B + 1)]


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation: forward D x dtype x dropout, main backward D x dtype x dropout x {default dQ, deterministic},
# the deterministic dQ kernel; 128-row backward tiles at D = 64, 64 rows at D = 128 and with dropout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["flat", "peaked"])
@pytest.mark.parametrize("p", [0.0, 0.17])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128])
def test_every_instantiation(D, dtype, p, regime):
    cu_q, cu_k = _fixed(2, 300, 300)
    _case(f"inst D={D} {str(dtype)[6:]} p={p} {regime}", cu_q, cu_k, 4, 2, D, dtype, True, (-1, -1), regime, p=p,
          dets=(False, True), seed=D + int(100 * p))


# ---------------------------------------------------------------------------------------------------------------------
# mask edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("diff", [-65, -1, 1, 63, 64, 65, 127, 129])
@pytest.mark.parametrize("window", [(-1, -1), (150, 0)])
@pytest.mark.parametrize("D", [64, 128])
def test_diagonal_alignment(D, window, diff):
    """Sk - Sq over residues of the 64- and 128-row tiles, causal and a causal window, with mask-probe logits: the
    backward's interior-tile test and the forward's interior skip see every alignment; Sq > Sk leaves rows without
    keys."""
    Sq = 300
    cu_q, cu_k = _fixed(2, Sq, Sq + diff)
    _case(f"align D={D} w={window} Sk-Sq={diff}", cu_q, cu_k, 2, 1, D, torch.bfloat16, True, window, "probe",
          dets=(False, True) if diff in (-65, 64) else (False,), seed=diff % 97)


@pytest.mark.parametrize("causal,window", [(False, (3, 0)), (False, (0, 5)), (False, (17, 9)), (True, (40, 0)),
                                           (False, (5, 40)), (False, (130, 129))])
@pytest.mark.parametrize("D", [64, 128])
def test_narrow_windows(D, causal, window):
    """Windows narrower than a tile, right > 0 and a window wider than one tile on each side."""
    cu_q, cu_k = _fixed(2, 333, 333)
    _case(f"window D={D} c={causal} w={window}", cu_q, cu_k, 2, 2, D, torch.bfloat16, causal, window, "probe",
          dets=(False, True), seed=window[0] + 7 * window[1])


@pytest.mark.parametrize("S", [1, 63, 65, 127, 129, 385])
@pytest.mark.parametrize("D", [64, 128])
def test_ragged_tails(D, S):
    """Sequences of S rows in a batch of 3: the last tile's rows past the sequence are the next sequence's."""
    cu_q, cu_k = _fixed(3, S, S)
    _case(f"tail D={D} S={S}", cu_q, cu_k, 2, 1, D, torch.bfloat16, True, (-1, -1), "probe", seed=S)
    _case(f"tail D={D} S={S} peaked non-causal", cu_q, cu_k, 2, 1, D, torch.float16, False, (-1, -1), "peaked",
          seed=S + 1)


@pytest.mark.parametrize("Hk", [8, 2, 1])
def test_gqa_groups(Hk):
    cu_q, cu_k = _fixed(2, 257, 257)
    for D in (64, 128):
        _case(f"gqa 8/{Hk} D={D}", cu_q, cu_k, 8, Hk, D, torch.bfloat16, True, (-1, -1), "peaked",
              dets=(False, True), seed=Hk)


@pytest.mark.parametrize("alibi_dims,scale", [(1, None), (2, None), (1, 0.3), (0, 0.3), (0, 0.02)])
@pytest.mark.parametrize("D", [64, 128])
def test_alibi_and_softmax_scale(D, alibi_dims, scale):
    """1-D ALiBi slopes (batch stride 0), 2-D slopes, and a non-default softmax_scale with and without ALiBi."""
    B, S, Hq, Hk = 2, 260, 4, 2
    cu_q, cu_k = _fixed(B, S, S + 30)
    gen = torch.Generator(device=DEV).manual_seed(D)
    alibi = None
    if alibi_dims:
        shape = (Hq,) if alibi_dims == 1 else (B, Hq)
        alibi = (0.02 + 0.3 * torch.rand(*shape, device=DEV, generator=gen)).float()
    for causal, regime in ((True, "peaked"), (False, "flat")):
        _case(f"alibi{alibi_dims} scale={scale} D={D} c={causal}", cu_q, cu_k, Hq, Hk, D, torch.bfloat16, causal,
              (-1, -1), regime, scale=scale, alibi=alibi, dets=(False, True), seed=alibi_dims + D)


@pytest.mark.parametrize("causal,window", [(True, (-1, -1)), (False, (-1, -1)), (True, (50, 0)), (False, (20, 30))])
def test_varlen_per_sequence_shift(causal, window):
    """cu_q != cu_k: each sequence has its own bottom-right shift, with empty query and empty key sequences, and
    sequences shorter than a tile; probe logits address packed key indices, so a key of a neighbouring sequence that
    leaked would dominate its row."""
    q_lens = [37, 0, 200, 5, 128, 0, 300, 64]
    k_lens = [100, 50, 0, 300, 1, 64, 129, 64]
    cu_q = [0] + list(torch.tensor(q_lens).cumsum(0).tolist())
    cu_k = [0] + list(torch.tensor(k_lens).cumsum(0).tolist())
    for D in (64, 128):
        _case(f"varlen D={D} c={causal} w={window}", cu_q, cu_k, 4, 2, D, torch.bfloat16, causal, window, "probe",
              dets=(False, True), seed=D)
    _case(f"varlen dropout c={causal} w={window}", cu_q, cu_k, 4, 2, 128, torch.float16, causal, window, "peaked",
          p=0.1, dets=(False, True), seed=3)


# ---------------------------------------------------------------------------------------------------------------------
# exact cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("diff", [0, 70, -3])
def test_window_zero_is_one_key(D, diff):
    """window (0, 0): each row sees exactly its diagonal key, so O is that key's V bitwise and the LSE is its scaled
    score within the fp32 dot product's error; rows before the first key (Sq > Sk) get O = 0, LSE = -inf."""
    Sq = 200
    cu_q, cu_k = _fixed(2, Sq, Sq + diff)
    R, runs = _case(f"window(0,0) D={D} Sk-Sq={diff}", cu_q, cu_k, 2, 2, D, torch.bfloat16, False, (0, 0), "peaked",
                    dets=(False, True), seed=diff + 5)
    o, lse = runs[False][:2]
    q3, k3, v3, _ = _make("peaked", cu_q, cu_k, 2, 2, D, torch.bfloat16, False, (0, 0), 1 / math.sqrt(D), diff + 5)
    for b in range(2):
        rows = torch.arange(Sq, device=DEV)
        key = rows + diff
        ok = key >= 0
        oq = o[cu_q[b]:cu_q[b + 1]]
        assert torch.equal(oq[ok], v3[cu_k[b] + key[ok]]), "O must be the one visible V, bitwise"
        assert bool((oq[~ok] == 0).all())
        s = (q3[cu_q[b]:cu_q[b + 1]][ok].double() * k3[cu_k[b] + key[ok]].double()).sum(-1) / math.sqrt(D)
        sabs = (q3[cu_q[b]:cu_q[b + 1]][ok].double().abs() * k3[cu_k[b] + key[ok]].double().abs()).sum(-1)
        lse_b = lse[:, cu_q[b]:cu_q[b + 1]].t()[ok]
        check(lse_b, s, f"window(0,0) D={D} Sk-Sq={diff} LSE = scale s", ulps=0,
              floor=D * U32 * sabs / math.sqrt(D) + 2.0 ** -21 * (s.abs() + 1), dtype=torch.float32)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal,window,diff", [(True, (-1, -1), 190), (True, (-1, -1), -40), (False, (77, 11), 0),
                                                (False, (-1, -1), 1)])
def test_zero_q_is_uniform(D, causal, window, diff):
    """q = 0: every visible key gets P = 1 exactly, so O is the mean of the visible V (within 1 ulp plus the fp32
    accumulation floor) and the LSE is ln(count) within fp32 rounding: a leaked or dropped key moves the LSE by at least
    ln((n + 1) / n) >= 1e-4."""
    Sq = 260
    cu_q, cu_k = _fixed(2, Sq, Sq + diff)
    R, runs = _case(f"q=0 D={D} c={causal} w={window} Sk-Sq={diff}", cu_q, cu_k, 4, 1, D, torch.bfloat16, causal,
                    window, "zero_q", dets=(False, True), seed=D + diff)
    o, lse = runs[False][:2]
    _, _, v3, _ = _make("zero_q", cu_q, cu_k, 4, 1, D, torch.bfloat16, causal, window, 1 / math.sqrt(D), D + diff)
    Sk = Sq + diff
    vis = _visible(Sq, Sk, causal, window).double()
    cnt = vis.sum(1)
    for b in range(2):
        vb = v3[cu_k[b]:cu_k[b + 1], 0].double()
        mean = (vis @ vb) / cnt.clamp(min=1)[:, None]
        floor = (Sk / 16 + Sk / 128 + 6) * 4 * U32 * (vis @ vb.abs()) / cnt.clamp(min=1)[:, None]
        ob = o[cu_q[b]:cu_q[b + 1]]
        for h in range(4):
            check(ob[:, h], mean, f"q=0 D={D} Sk-Sq={diff} O = mean V", floor=floor)
        lref = torch.where(cnt > 0, cnt.log(), -math.inf)
        lb = lse[:, cu_q[b]:cu_q[b + 1]]
        fin = cnt > 0
        assert bool((lb[:, ~fin] == -math.inf).all())
        check(lb[:, fin], lref[fin].expand(4, -1), f"q=0 D={D} Sk-Sq={diff} LSE = ln(count)", ulps=0,
              floor=2.0 ** -21 * (lref[fin].abs() + 1), dtype=torch.float32)


# ---------------------------------------------------------------------------------------------------------------------
# the fused-QKV fast path and the flagship shape
# ---------------------------------------------------------------------------------------------------------------------
def _run_qkvpacked(B, S, hq, hk, D, regime, det, cu=None, seed=0):
    from torchacc_b200.ops import attention as A
    cu_l = cu if cu is not None else [b * S for b in range(B + 1)]
    scale = 1.0 / math.sqrt(D)
    q3, k3, v3, do3 = _make(regime, cu_l, cu_l, hq, hk, D, torch.bfloat16, True, (-1, -1), scale, seed)
    T = cu_l[-1]
    qkv = torch.cat([q3.reshape(T, -1), k3.reshape(T, -1), v3.reshape(T, -1)], 1).requires_grad_()
    A.set_deterministic(det)
    try:
        if cu is None:
            out = A.flash_attn_qkvpacked_tokens(qkv, hq, hk, D, B, S, causal=True)
        else:   # a packed batch as the native Llama passes it: batch 1, seq_len T, the sequences in cu_seqlens
            out = A.flash_attn_qkvpacked_tokens(qkv, hq, hk, D, 1, T, causal=True,
                                                cu_seqlens=torch.tensor(cu, dtype=torch.int32, device=DEV))
        out.backward(do3.reshape(T, -1))
    finally:
        A.set_deterministic(False)
    o = out.detach().view(T, hq, D)
    g = qkv.grad
    dq = g[:, :hq * D].view(T, hq, D)
    dk = g[:, hq * D:(hq + hk) * D].view(T, hk, D)
    dv = g[:, (hq + hk) * D:].view(T, hk, D)
    return (q3, k3, v3, do3), cu_l, o, dq, dk, dv


@pytest.mark.parametrize("packed", [False, True])
def test_qkvpacked_strided_views(packed):
    """flash_attn_qkvpacked_tokens reads q / k / v as strided column blocks of one [T, (Hq + 2 Hk) D] activation and
    writes dQ / dK / dV into one buffer; fixed-length and cu_seqlens-packed."""
    cu = [0, 100, 356, 361, 700] if packed else None
    for det in (False, True):
        (q3, k3, v3, do3), cu_l, o, dq, dk, dv = _run_qkvpacked(2, 350, 8, 2, 128, "peaked", det, cu, seed=11)
        R = _reference(q3, k3, v3, do3, o, None, cu_l, cu_l, 1 / math.sqrt(128), True, (-1, -1))
        _check_fwd(f"qkvpacked packed={packed} det={det}", R, o)
        _check_bwd(f"qkvpacked packed={packed} det={det}", R, dq, dk, dv)


def test_flagship_shape_all_heads():
    """B = 2, S = 4096, 32 query / 8 KV heads, D = 128, causal through flash_attn_qkvpacked_tokens (the bench
    workload), forward and backward against fp64 on every head."""
    (q3, k3, v3, do3), cu_l, o, dq, dk, dv = _run_qkvpacked(2, 4096, 32, 8, 128, "flat", False, seed=1)
    R = _reference(q3, k3, v3, do3, o, None, cu_l, cu_l, 1 / math.sqrt(128), True, (-1, -1))
    _check_fwd("flagship", R, o)
    _check_bwd("flagship", R, dq, dk, dv)


def test_long_sequence_peaked():
    """S = 8192 (64 key tiles per row at the end of the sequence) with peaked logits, both backward paths."""
    cu_q, cu_k = _fixed(1, 8192, 8192)
    _case("S=8192 peaked", cu_q, cu_k, 2, 1, 128, torch.bfloat16, True, (-1, -1), "peaked", dets=(False, True), seed=2)


# ---------------------------------------------------------------------------------------------------------------------
# blockwise (ring) kernels: in-kernel LSE merge (acc_init 1 and 0), zigzag half-block views, phased backward
# ---------------------------------------------------------------------------------------------------------------------
def _shard(x, r, cp):
    c = x.chunk(2 * cp, dim=1)
    return torch.cat([c[r], c[2 * cp - 1 - r]], 1).contiguous()


def _unshard(parts, cp):
    chunks = [None] * (2 * cp)
    for r, p in enumerate(parts):
        a, b = p.chunk(2, dim=1)
        chunks[r], chunks[2 * cp - 1 - r] = a, b
    return torch.cat(chunks, 1)


@pytest.mark.parametrize("regime", ["flat", "peaked"])
@pytest.mark.parametrize("cp,D", [(2, 128), (4, 128), (4, 64)])
def test_ring_blockwise_matches_fp64(cp, D, regime):
    """ring_forward_native / ring_backward_native, causal zigzag, every rank simulated on one GPU, against one
    full-sequence fp64 attention: O and the merged LSE under the merge bound, dQ / dK / dV summed over the ranks."""
    from torchacc_b200.ops.context_parallel import ring as R_
    B, S, Hq, Hk = 2, 1536, 4, 2
    scale = 1.0 / math.sqrt(D)
    cu = [b * S for b in range(B + 1)]
    q3, k3, v3, do3 = _make(regime, cu, cu, Hq, Hk, D, torch.bfloat16, True, (-1, -1), scale, cp + D)
    q, k, v, do = (t.view(B, S, -1, D) for t in (q3, k3, v3, do3))
    blocks = [torch.stack([_shard(k, j, cp), _shard(v, j, cp)], 0) for j in range(cp)]
    outs, lses, dqs, dkv_sum = [], [], [], None
    for r in range(cp):
        steps = R_._plan(r, cp, True, True)
        q_r, do_r = _shard(q, r, cp), _shard(do, r, cp)
        out_r, lse_r = R_.ring_forward_native(q_r, blocks, steps, scale)
        dq_r, dkv_r = R_.ring_backward_native(do_r, q_r, out_r, lse_r, blocks, steps, scale)
        outs.append(out_r)
        lses.append(lse_r.view(Hq, B, -1).permute(1, 2, 0))
        dqs.append(dq_r)
        dkv_sum = dkv_r.double() if dkv_sum is None else dkv_sum + dkv_r.double()
    o = _unshard(outs, cp).reshape(B * S, Hq, D)
    lse = _unshard(lses, cp).permute(2, 0, 1).reshape(Hq, B * S)
    dq = _unshard(dqs, cp).reshape(B * S, Hq, D)
    dk = _unshard([dkv_sum[j, 0] for j in range(cp)], cp).reshape(B * S, Hk, D)
    dv = _unshard([dkv_sum[j, 1] for j in range(cp)], cp).reshape(B * S, Hk, D)
    R = _reference(q3, k3, v3, do3, o, lse, cu, cu, scale, True, (-1, -1), blocks=cp)
    tag = f"ring cp={cp} D={D} {regime}"
    _check_fwd(tag, R, o, lse)
    # dK / dV are fp32 sums of the ranks' 16-bit contributions: their roundings are in the floor, not in an ulp term
    check(dq, R["dq"], f"{tag} dQ", floor=(1 + 2.0 ** -8) * R["bdq"])
    check(dk, R["dk"], f"{tag} dK", ulps=0, floor=(1 + 2.0 ** -8) * R["bdk"], dtype=torch.bfloat16)
    check(dv, R["dv"], f"{tag} dV", ulps=0, floor=(1 + 2.0 ** -8) * R["bdv"], dtype=torch.bfloat16)
