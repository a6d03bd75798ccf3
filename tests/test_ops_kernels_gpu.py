"""The bandwidth-bound op kernels (csrc/ops/norm_rope_act.cu, csrc/ops/loss_optim.cu) at the flagship shapes and at
their numeric edges, against fp64 PyTorch references of the same math computed from the exact 16-bit inputs.

Shapes are chosen so that every launch variant and loop branch runs: every RMSNorm forward ``kVpt`` and backward
(threads, vpt) pair, more rows than CTAs (grid-stride row loops, backward next-row prefetch), SwiGLU's second vector
pair (F > 2048), RoPE's grid-stride loop, the cross-entropy tail loop, AdamW's second 16-byte group per trip.

Tolerances are in units of the output dtype (``ulp_err``), plus, where a result comes out of a reduction or a
cancellation, a floor derived from the fp32 arithmetic that produces it (derivations next to each bound)."""
import functools
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
LLAMA3_SCALING = {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                  "original_max_position_embeddings": 8192}


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def ulp_dtype(ref64, dtype):
    """Spacing of ``dtype`` at |ref| (2^floor(log2 |ref|) * eps); below the smallest normal number, the subnormal
    spacing, so results that flush to (or round among) subnormals are held to that fixed floor."""
    fi = torch.finfo(dtype)
    return torch.exp2(torch.floor(torch.log2(ref64.abs().clamp(min=fi.tiny)))) * fi.eps


def ulp_err(out, ref64, dtype):
    """|out - ref| / ulp_dtype(|ref|), elementwise."""
    return (out.double() - ref64).abs() / ulp_dtype(ref64, dtype)


def check(out, ref64, what, ulps=1.0, floor=None, dtype=None):
    """Every element within ``ulps`` ulps of the fp64 reference, plus ``floor`` (absolute, broadcastable).  NaN in
    the output fails.  Prints and returns the largest ulp error seen."""
    dtype = dtype or out.dtype
    err = (out.double() - ref64).abs()
    u = ulp_dtype(ref64, dtype)
    tol = ulps * u + (0.0 if floor is None else floor)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} outside {ulps} ulp + floor; first at flat index "
                             f"{i}: out {out.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r} "
                             f"tol {tol.reshape(-1)[i].item() if tol.dim() else float(tol):.3g}")
    worst = float(ulp_err(out, ref64, dtype).max()) if out.numel() else 0.0
    used = float((err / tol).max()) if out.numel() else 0.0
    print(f"[ulp] {what}: max {worst:.3f} ulp, {used:.3f} of the bound")
    return worst


@functools.lru_cache(maxsize=None)
def _tables(D):
    from torchacc_b200.ops.rope import rope_tables
    return rope_tables(131072, D, theta=500000.0, device=DEV, scaling=LLAMA3_SCALING)


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm
# ---------------------------------------------------------------------------------------------------------------------
def _rmsnorm_inputs(rows, H, dtype, gen):
    x = torch.randn(rows, H, device=DEV, generator=gen)
    if rows >= 3:
        x[0] = 0.0                                                                       # all-zero row
        x[1] = 3.0e4 * torch.sign(torch.randn(H, device=DEV, generator=gen))             # +-3e4 (fp16-safe)
        x[2] = 1e-2 * x[2]
        x[2, H // 3] = 1.0e3                                                             # one dominant element
    return x.to(dtype)


def _run_rmsnorm(rows, H, dtype, mode, seed=0):
    from torchacc_b200.ops.rmsnorm import rmsnorm
    gen = torch.Generator(device=DEV).manual_seed(seed)
    eps = 1e-5
    x = _rmsnorm_inputs(rows, H, dtype, gen).requires_grad_()
    w = (1 + 0.1 * torch.randn(H, device=DEV, generator=gen)).to(dtype).requires_grad_()
    res = torch.randn(rows, H, device=DEV, generator=gen).to(dtype).requires_grad_() if mode == "residual" else None
    dy = torch.randn(rows, H, device=DEV, generator=gen).to(dtype)
    dh = torch.randn(rows, H, device=DEV, generator=gen).to(dtype)
    y, h = rmsnorm(x, w, eps, residual=res, passthrough=(mode == "passthrough"))
    outs, grads = [y], [dy]
    if h is not None:
        outs.append(h)
        grads.append(dh)
    torch.autograd.backward(outs, grads)

    # forward: the kernel normalises the residual stream exactly as stored (fp32 add, rounded to the dtype)
    if mode == "residual":
        h_ref = (x.detach().float() + res.detach().float()).to(dtype)
        assert torch.equal(h, h_ref), "h = x + residual is not the rounded fp32 sum"
    else:
        h_ref = x.detach()
        if mode == "passthrough":
            assert torch.equal(h, h_ref)
    h64, w64, dy64 = h_ref.double(), w.detach().double(), dy.double()
    rs64 = torch.rsqrt(h64.square().mean(-1, keepdim=True) + eps)
    xh = h64 * rs64
    # y = h * rstd * w: elementwise after a well-conditioned sum of squares (relative error of rstd ~ 1e-7), so
    # one rounding to the dtype, at most 1 ulp
    check(y.detach(), xh * w64, f"rmsnorm y H={H} {dtype} {mode} rows={rows}")

    # backward: dx = rstd (dy w - xhat mean(dy w xhat)) [+ dres].  The mean is an fp32 sum of H terms (a few dozen
    # sequential adds per thread, then a tree: relative error <~ 1e-6 of sum |dy w xhat| / H), and dx cancels two
    # terms: floor 1e-5 x the row's largest |rstd dy w| + |xhat mean|-scale term, i.e. 1e-5 x max |ref| of the row
    # computed without cancellation.
    gw = dy64 * w64
    dot = (gw * xh).mean(-1, keepdim=True)
    dx64 = rs64 * (gw - xh * dot)
    if mode != "plain":
        dx64 = dx64 + dh.double()
    scale_row = (rs64 * (gw.abs() + (xh * dot).abs())).amax(-1, keepdim=True)
    check(x.grad, dx64, f"rmsnorm dx H={H} {dtype} {mode} rows={rows}", floor=1e-5 * scale_row)
    if mode == "residual":
        assert torch.equal(res.grad, x.grad)
    # dw: fp32 per-CTA partial column sums (<= 32 rows each at these shapes) summed over <= 264 partials in fp32, then
    # rounded to the dtype: floor 1e-5 x sum over rows of |dy xhat| (rounding errors of ~300 sequential fp32 adds stay
    # well inside 2^-24 x 300 ~ 2e-5 and in practice grow like its square root)
    dw64 = (dy64 * xh).sum(0)
    check(w.grad, dw64, f"rmsnorm dw H={H} {dtype} {mode} rows={rows}", floor=1e-5 * (dy64 * xh).abs().sum(0))


@pytest.mark.parametrize("mode", ["plain", "residual", "passthrough"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("H", [2304, 3072, 4096, 5120, 8192, 12288, 16384])
def test_rmsnorm_matches_fp64(H, dtype, mode):
    """1057 rows: one more than the forward grid (8 CTAs x 132 SMs), four times the backward's 264 CTAs.  The H values
    reach forward kVpt 2 / 4 / 8 and backward (256 threads, vpt 2), (512, 1), (512, 2), (512, 4)."""
    _run_rmsnorm(1057, H, dtype, mode)


@pytest.mark.parametrize("mode", ["residual", "passthrough"])
@pytest.mark.parametrize("H", [4096, 12288])
@pytest.mark.parametrize("rows", [1, 7, 8192])
def test_rmsnorm_row_counts(rows, H, mode):
    """Fewer rows than CTAs (one row per CTA, no prefetch) and the flagship 8192 rows (8 rows per forward CTA, 31 per
    backward CTA, so the next-row prefetch runs on every trip)."""
    _run_rmsnorm(rows, H, torch.bfloat16, mode, seed=rows)


# ---------------------------------------------------------------------------------------------------------------------
# RoPE
# ---------------------------------------------------------------------------------------------------------------------
def _rope_ref(x64, c64, s64, sign):
    """x64 [T, h, D]; c64 / s64 [T, 1, D/2] (the kernel's fp32 tables, in fp64).  Returns the rotated fp64 tensor and
    the sum of the magnitudes of the two products per output element (scale of the fp32 cancellation)."""
    half = x64.shape[-1] // 2
    x1, x2 = x64[..., :half], x64[..., half:]
    s = s64 * sign
    out = torch.cat([x1 * c64 - x2 * s, x2 * c64 + x1 * s], -1)
    mag = torch.cat([(x1 * c64).abs() + (x2 * s).abs(), (x2 * c64).abs() + (x1 * s).abs()], -1)
    return out, mag


def _check_rope(out, ref, mag, what):
    # each output is a*c -/+ b*s in fp32 (two products, one add, possibly fused): error <= 2^-23 (|a c| + |b s|) before
    # the final rounding, so 1 ulp plus that floor, which only matters where the two products cancel
    return check(out, ref, what, floor=2.0 ** -22 * mag)


def _positions(T, B, pos_mode, gen):
    if pos_mode == "seq":
        return None, T // B, torch.arange(T, device=DEV) % (T // B)
    pos = torch.randint(0, 131072, (T,), device=DEV, generator=gen, dtype=torch.int32)
    pos[0], pos[-1], pos[T // 2] = 131071, 0, 131071                       # the table's last row, and its first
    return pos, 131072, pos.long()


@pytest.mark.parametrize("pos_mode", ["seq", "positions"])
@pytest.mark.parametrize("entry", ["rope_qkv_", "apply_rope", "rope_one"])
@pytest.mark.parametrize("heads", [(32, 8), (8, 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_rope_matches_fp64(D, dtype, heads, entry, pos_mode):
    _run_rope(D, dtype, heads, entry, pos_mode, B=3, S=97)


def test_rope_grid_stride_loop():
    """T = 8192, 40 heads, D = 128: 8192 x 40 x 8 vectors > 16 CTAs/SM x 132 SMs x 256 threads, so the loop strides."""
    _run_rope(128, torch.bfloat16, (32, 8), "rope_qkv_", "positions", B=2, S=4096)


def _run_rope(D, dtype, heads, entry, pos_mode, B, S):
    from torchacc_b200.ops.rope import _RopeOneFn, apply_rope, rope_qkv_
    hq, hk = heads
    T = B * S
    gen = torch.Generator(device=DEV).manual_seed(D + hq)
    cos, sin = _tables(D)
    positions, seq_len, pos_long = _positions(T, B, pos_mode, gen)
    c64, s64 = cos[pos_long].double().unsqueeze(1), sin[pos_long].double().unsqueeze(1)
    W = (hq + 2 * hk) * D
    base = torch.randn(T, W, device=DEV, generator=gen).to(dtype).requires_grad_()
    gout = torch.randn(T, W, device=DEV, generator=gen).to(dtype)
    tag = f"rope D={D} {dtype} {hq}/{hk} {entry} {pos_mode}"
    if entry == "rope_qkv_":
        qkv = base.clone()
        out = rope_qkv_(qkv, hq, hk, D, cos, sin, positions, seq_len)
        q_out, k_out, v_out = out[:, :hq * D], out[:, hq * D:(hq + hk) * D], out[:, (hq + hk) * D:]
        out.backward(gout)
        dbase = base.grad
    elif entry == "apply_rope":
        # q and k as separate strided (non-view) buffers whose token pitches differ from each other and from D*h
        qs = torch.empty_strided((T, hq, D), ((hq * D + 64), D, 1), dtype=dtype, device=DEV)
        ks = torch.empty_strided((T, hk, D), ((hk * D + 136), D, 1), dtype=dtype, device=DEV)
        qs.copy_(base[:, :hq * D].view(T, hq, D))
        ks.copy_(base[:, hq * D:(hq + hk) * D].view(T, hk, D))
        qo, ko = apply_rope(qs, ks, cos, sin, positions, seq_len)
        q_out, k_out, v_out = qo.reshape(T, -1), ko.reshape(T, -1), base[:, (hq + hk) * D:].detach()
        torch.autograd.backward([qo, ko], [gout[:, :hq * D].view(T, hq, D), gout[:, hq * D:(hq + hk) * D].view(T, hk, D)])
        dbase = base.grad
    else:
        # the HF path: one tensor at a time, each a strided view of the projection output
        proj = base.clone()
        qv = proj[:, :hq * D].view(T, hq, D)
        qo = _RopeOneFn.apply(qv, cos, sin, positions, seq_len)
        kv = proj[:, hq * D:(hq + hk) * D].view(T, hk, D)
        ko = _RopeOneFn.apply(kv, cos, sin, positions, seq_len)
        q_out, k_out, v_out = qo.reshape(T, -1), ko.reshape(T, -1), proj[:, (hq + hk) * D:]
        torch.autograd.backward([qo, ko, v_out], [gout[:, :hq * D].view(T, hq, D),
                                                  gout[:, hq * D:(hq + hk) * D].view(T, hk, D), gout[:, (hq + hk) * D:]])
        dbase = base.grad
    x64 = base.detach().double()
    q_ref, q_mag = _rope_ref(x64[:, :hq * D].view(T, hq, D), c64, s64, 1.0)
    k_ref, k_mag = _rope_ref(x64[:, hq * D:(hq + hk) * D].view(T, hk, D), c64, s64, 1.0)
    _check_rope(q_out.detach().reshape(T, hq, D), q_ref, q_mag, f"{tag} q")
    _check_rope(k_out.detach().reshape(T, hk, D), k_ref, k_mag, f"{tag} k")
    assert torch.equal(v_out.detach(), base.detach()[:, (hq + hk) * D:]), f"{tag}: V was modified"
    g64 = gout.double()
    dq_ref, dq_mag = _rope_ref(g64[:, :hq * D].view(T, hq, D), c64, s64, -1.0)
    dk_ref, dk_mag = _rope_ref(g64[:, hq * D:(hq + hk) * D].view(T, hk, D), c64, s64, -1.0)
    _check_rope(dbase[:, :hq * D].view(T, hq, D), dq_ref, dq_mag, f"{tag} dq")
    _check_rope(dbase[:, hq * D:(hq + hk) * D].view(T, hk, D), dk_ref, dk_mag, f"{tag} dk")
    if entry != "apply_rope":
        assert torch.equal(dbase[:, (hq + hk) * D:], gout[:, (hq + hk) * D:]), f"{tag}: dV is not the incoming gradient"


# ---------------------------------------------------------------------------------------------------------------------
# SwiGLU
# ---------------------------------------------------------------------------------------------------------------------
def _silu_ref(g64):
    s = torch.sigmoid(g64)
    return s, g64 * s


def _check_swiglu(h, dg, du, g64, u64, dh64, tag, dtype):
    """h = silu(g) u and du = dh silu(g) are products of well-conditioned factors: the kernel's sigmoid has a relative
    error of a few 2^-22 (MUFU ex2 + rcp, plus the rounding of x log2 e: <= 2^-24 |x| log2 e relative, 3.4e-6 at
    |x| = 40) far below half an ulp of a 16-bit type, so at most 1 ulp.  dg = dh u (s + silu (1 - s)) has a root near
    g = -1.28 where its two terms cancel: floor 2^-18 |dh u| (|s| + |silu (1 - s)|).  Observed on an H100 over every
    shape of the swiglu tests: h and du at most 0.501 ulp, dg within 0.50 of its bound."""
    s, silu = _silu_ref(g64)
    worst = {}
    if h is not None:
        worst["h"] = check(h, silu * u64, f"{tag} h", dtype=dtype)
    if du is not None:
        worst["du"] = check(du, dh64 * silu, f"{tag} du", dtype=dtype)
    if dg is not None:
        mag = (dh64 * u64).abs() * (s.abs() + (silu * (1 - s)).abs())
        worst["dg"] = check(dg, dh64 * u64 * (s + silu * (1 - s)), f"{tag} dg", floor=2.0 ** -18 * mag, dtype=dtype)
    return worst


def _swiglu_inputs(T, Fd, dtype, gen):
    g = (3 * torch.randn(T, Fd, device=DEV, generator=gen)).to(dtype)
    u = torch.randn(T, Fd, device=DEV, generator=gen).to(dtype)
    dh = torch.randn(T, Fd, device=DEV, generator=gen).to(dtype)
    return g, u, dh


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("T", [300, 1057, 8192])
@pytest.mark.parametrize("Fd", [1408, 2816, 14336])
def test_swiglu_matches_fp64(Fd, T, dtype):
    """F > 2048 runs the second vector pair (v + 256) of every 512-vector trip; T > 1056 makes the row loop stride."""
    from torchacc_b200.ops.swiglu import swiglu, swiglu_separate
    gen = torch.Generator(device=DEV).manual_seed(Fd + T)
    g, u, dh = _swiglu_inputs(T, Fd, dtype, gen)
    g64, u64, dh64 = g.double(), u.double(), dh.double()
    # fused gate|up input [T, 2F]
    gu = torch.cat([g, u], 1).requires_grad_()
    h = swiglu(gu)
    h.backward(dh)
    _check_swiglu(h.detach(), gu.grad[:, :Fd], gu.grad[:, Fd:], g64, u64, dh64, f"swiglu F={Fd} T={T} {dtype}", dtype)
    del gu, h
    # separate strided g / u views, distinct pitches (F + 16 and F + 40, u starting 8 elements in)
    gbuf = torch.zeros(T, Fd + 16, device=DEV, dtype=dtype)
    ubuf = torch.zeros(T, Fd + 40, device=DEV, dtype=dtype)
    gbuf[:, :Fd] = g
    ubuf[:, 8:Fd + 8] = u
    gbuf.requires_grad_()
    ubuf.requires_grad_()
    gv, uv = gbuf[:, :Fd], ubuf[:, 8:Fd + 8]
    assert gv.stride(0) == Fd + 16 and uv.stride(0) == Fd + 40
    h2 = swiglu_separate(gv, uv)
    h2.backward(dh)
    _check_swiglu(h2.detach(), gbuf.grad[:, :Fd], ubuf.grad[:, 8:Fd + 8], g64, u64, dh64,
                  f"swiglu_separate F={Fd} T={T} {dtype}", dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("T", [300, 1057, 8192])
@pytest.mark.parametrize("Fd", [1408, 2816, 14336])
def test_gate_up_swiglu_matches_fp64(Fd, T, dtype):
    """The GEMM epilogue applies the sigmoid to the fp32 accumulators.  x and W hold multiples of 1/8 in [-1, 1] and
    K = 64, so every product and partial sum is exact in fp32: g and u are exact and h is held to 1 ulp.  The
    backward's GEMMs take the swiglu_bwd output rounded to the dtype: |d(dx)| <= 1 ulp + 2^-eps_bits (|dgu| @ |W|)."""
    from torchacc_b200.ops.swiglu import gate_up_swiglu
    gen = torch.Generator(device=DEV).manual_seed(Fd * T)
    K = 64
    x = (torch.randint(-8, 9, (T, K), device=DEV, generator=gen) / 8).to(dtype).requires_grad_()
    w = (torch.randint(-8, 9, (2 * Fd, K), device=DEV, generator=gen) / 8).to(dtype).requires_grad_()
    dh = torch.randn(T, Fd, device=DEV, generator=gen).to(dtype)
    h = gate_up_swiglu(x, w)
    h.backward(dh)
    gu64 = x.detach().double() @ w.detach().double().t()
    g64, u64, dh64 = gu64[:, :Fd], gu64[:, Fd:], dh.double()
    _check_swiglu(h.detach(), None, None, g64, u64, dh64, f"gate_up_swiglu F={Fd} T={T} {dtype}", dtype)
    s, silu = _silu_ref(g64)
    dgu64 = torch.cat([dh64 * u64 * (s + silu * (1 - s)), dh64 * silu], 1)
    eps = torch.finfo(dtype).eps
    check(x.grad, dgu64 @ w.detach().double(), f"gate_up_swiglu dx F={Fd} T={T} {dtype}",
          floor=eps * (dgu64.abs() @ w.detach().double().abs()))
    check(w.grad, dgu64.t() @ x.detach().double(), f"gate_up_swiglu dw F={Fd} T={T} {dtype}",
          floor=eps * (dgu64.abs().t() @ x.detach().double().abs()))


def _all_bf16_in(lo, hi):
    """Every bf16 value in [lo, hi] (both signs of zero excluded but one), as a bf16 tensor on the GPU."""
    bits = torch.arange(0, 1 << 16, dtype=torch.int32, device=DEV).to(torch.int16).view(torch.bfloat16)
    v = bits[torch.isfinite(bits) & (bits >= lo) & (bits <= hi)]
    return v[~((v == 0) & torch.signbit(v))]


def test_swiglu_sigmoid_exhaustive_bf16():
    """silu and its derivative at every bf16 g in [-40, 40], u = dh = 1, through the swiglu kernels and both sites of
    the GEMM epilogue.  The reference is the fp64 sigmoid, so the kernel's sigmoid must keep its relative accuracy for
    negative g, where sigmoid(g) is tiny.  Observed on an H100 with the ex2 + rcp sigmoid: h, du and dg at most 0.50
    ulp at all three sites.  The former 0.5 + 0.5 tanh.approx(g / 2) form broke the 1-ulp bound at 223 of the 34816
    values in the swiglu kernel (silu(-7.8) came out as -0.001457 instead of -0.001465, 5 ulp)."""
    from torchacc_b200.ops.swiglu import gate_up_swiglu, swiglu
    g = _all_bf16_in(-40.0, 40.0)
    n = g.numel()
    cols = 256
    rows = -(-n // cols // 8) * 8                                         # the epilogue GEMM below takes K = rows
    gm = torch.zeros(rows * cols, dtype=torch.bfloat16, device=DEV)
    gm[:n] = g
    gm = gm.view(rows, cols)
    ones = torch.ones_like(gm)
    gu = torch.cat([gm, ones], 1).requires_grad_()
    h = swiglu(gu)
    h.backward(ones)
    g64 = gm.double()
    _check_swiglu(h.detach(), gu.grad[:, :cols], gu.grad[:, cols:], g64, ones.double(), ones.double(),
                  "sigmoid sweep swiglu", torch.bfloat16)
    # the epilogue: x = identity, so the accumulator of output (t, f) is exactly W_gate[f, t] = g[t, f].  Subnormal
    # g are left out: the tensor cores flush them before the epilogue sees them.
    ge = torch.where(gm.float().abs() < torch.finfo(torch.float32).tiny, torch.zeros_like(gm), gm)
    x = torch.eye(rows, dtype=torch.bfloat16, device=DEV)
    w = torch.cat([ge.t(), ones.t()], 0).contiguous()                     # [2F, K = rows]
    for write_gu in (False, True):
        xx = x.clone().requires_grad_(write_gu)                          # with a grad the GEMM also stores g|u
        hh = gate_up_swiglu(xx, w)
        _check_swiglu(hh.detach(), None, None, ge.double(), ones.double(), ones.double(),
                      f"sigmoid sweep epilogue write_gu={write_gu}", torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------------------
# Cross-entropy
# ---------------------------------------------------------------------------------------------------------------------
def _ce_ref(logits, labels, ignore_index=-100):
    """fp64 per-row loss, lse and softmax - onehot (0 rows for ignored labels) of bf16 logits [n, V]."""
    l64 = logits.double()
    lse = torch.logsumexp(l64, -1)
    valid = labels != ignore_index
    lab = labels.clamp(min=0)
    rows = torch.where(valid, lse - l64.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    p = torch.exp(l64 - lse[:, None])
    onehot = torch.zeros_like(p).scatter_(1, lab[:, None], 1.0)
    grad = torch.where(valid[:, None], p - onehot, torch.zeros_like(p))
    return rows, lse, grad, p, onehot


def _check_ce_grad(grad, p, onehot, grad_ref, gscale, what):
    """Each element is (exp2((f - max) log2 e) / sum - onehot) x scale in fp32.  ex2.approx is within 2 ulp, and the
    rounding of (f - max) log2 e adds 2^-24 |f - max| log2 e ln 2 relative (<= 1e-5 for |f - max| <= 128); the sum
    of exps adds ~2e-6: floor gscale (2e-5 p + 2^-23) (the 2^-23 covers the rounding of p - 1 at the label).
    Observed on an H100 over every cross-entropy test: at most 0.54 ulp, 0.54 of the bound."""
    return check(grad, grad_ref * gscale, what, floor=gscale * (2e-5 * p + 2.0 ** -23 * onehot))


def _check_ce_loss(loss, rows_ref, lse, scale, what):
    """Per row lse - logit = max + log(sum) - logit in fp32: the sum's ~1e-5 relative error is ~1e-5 absolute after
    the log, and max + log rounds at 2^-24 |lse|; the rows are then summed in fp32 (torch)."""
    ref = rows_ref.sum() * scale
    floor = scale * (1e-5 + 2.0 ** -23 * lse.abs()).sum()
    return check(loss.detach().reshape(()), ref, what, floor=floor, dtype=torch.float32)


def _labels(n, V, gen, ignore_frac=0.1):
    lab = torch.randint(0, V, (n,), device=DEV, generator=gen)
    if n >= 4:
        lab[0], lab[1], lab[2] = 0, V - 1, V - 3              # first logit, last logit, last vector
        drop = torch.rand(n, device=DEV, generator=gen) < ignore_frac
        drop[:3] = False
        lab[drop] = -100
    return lab


@pytest.mark.parametrize("reduction", ["mean", "sum"])
@pytest.mark.parametrize("n", [1, 300, 2048])
@pytest.mark.parametrize("V", [32000, 50304, 128256, 151936])
def test_cross_entropy_matches_fp64(V, n, reduction):
    from torchacc_b200.ops.cross_entropy import cross_entropy
    gen = torch.Generator(device=DEV).manual_seed(V + n)
    # spread +-60: exp of the smallest logits underflows relative to the largest, the lse sits near the max
    logits = (torch.rand(n, V, device=DEV, generator=gen) * 120 - 60).bfloat16().requires_grad_()
    lab = _labels(n, V, gen)
    loss = cross_entropy(logits, lab, reduction=reduction)
    loss.backward()
    rows, lse, g, p, onehot = _ce_ref(logits.detach(), lab)
    nv = max(int((lab != -100).sum()), 1)
    scale = 1.0 / nv if reduction == "mean" else 1.0
    _check_ce_loss(loss, rows, lse, scale, f"ce loss V={V} n={n} {reduction}")
    _check_ce_grad(logits.grad, p, onehot, g, scale, f"ce grad V={V} n={n} {reduction}")


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_cross_entropy_all_rows_ignored(reduction):
    from torchacc_b200.ops.cross_entropy import cross_entropy
    logits = torch.randn(64, 128256, device=DEV).bfloat16().requires_grad_()
    lab = torch.full((64,), -100, device=DEV, dtype=torch.long)
    loss = cross_entropy(logits, lab, reduction=reduction)
    loss.backward()
    assert float(loss) == 0.0
    assert bool((logits.grad == 0).all()), "ignored rows must have an exactly zero gradient"


@pytest.mark.parametrize("mask", ["first64", "half"])
@pytest.mark.parametrize("V", [32000, 128256])
def test_cross_entropy_masked_logits(V, mask):
    """-inf logits (masked vocabulary).  With the first 64 logits masked, threads 0-7 start on an all -inf vector and
    see finite logits on their next trip; with a random half masked, some of the 1024 threads do the same.  The online
    max / sum update must not compute (-inf) - (-inf)."""
    from torchacc_b200.ops.cross_entropy import cross_entropy
    gen = torch.Generator(device=DEV).manual_seed(V)
    n = 64
    logits = torch.randn(n, V, device=DEV, generator=gen) * 4
    if mask == "first64":
        masked = torch.zeros(n, V, dtype=torch.bool, device=DEV)
        masked[:, :64] = True
    else:
        masked = torch.rand(n, V, device=DEV, generator=gen) < 0.5
    logits[masked] = -math.inf
    logits = logits.bfloat16()
    # labels on unmasked logits
    lab = torch.multinomial((~masked).float(), 1, generator=gen)[:, 0]
    lg = logits.clone().requires_grad_()
    loss = cross_entropy(lg, lab)
    loss.backward()
    assert math.isfinite(float(loss)), f"loss {float(loss)} with masked logits"
    rows, lse, g, p, onehot = _ce_ref(logits, lab)
    _check_ce_loss(loss, rows, lse, 1.0 / n, f"ce masked {mask} V={V} loss")
    _check_ce_grad(lg.grad, p, onehot, g, 1.0 / n, f"ce masked {mask} V={V} grad")
    assert bool((lg.grad[masked] == 0).all())


@pytest.mark.parametrize("V", [50257, 32001])
def test_cross_entropy_tail_loop(V):
    """V % 8 != 0 on a [:, :V] view of a buffer whose pitch is padded to a multiple of 8: the scalar tail loop runs
    (label V - 1 sits in it), per-row losses are checked, and the padding columns stay untouched."""
    from torchacc_b200.ops.cross_entropy import _ce_native
    gen = torch.Generator(device=DEV).manual_seed(V)
    n = 257
    pitch = (V + 7) // 8 * 8 + 8
    buf = (torch.rand(n, pitch, device=DEV, generator=gen) * 40 - 20).bfloat16()
    lg = buf[:, :V]
    assert lg.stride(0) == pitch
    lab = _labels(n, V, gen)
    lab[3] = V - 2
    logits = lg.clone()
    pad = buf[:, V:].clone()
    scale = torch.full((1,), 1.0 / 200, device=DEV)
    rows = _ce_native(lg, lab, -100, scale, True)
    rows_ref, lse, g, p, onehot = _ce_ref(logits, lab)
    # per row: ~1e-5 from the sum and the log, 2^-24 |lse| from max + log
    check(rows, rows_ref, f"ce tail V={V} rows", floor=1e-5 + 2.0 ** -23 * lse.abs(), dtype=torch.float32)
    _check_ce_grad(lg, p, onehot, g, 1.0 / 200, f"ce tail V={V} grad")
    assert torch.equal(buf[:, V:], pad), "the kernel wrote past column V"


@pytest.mark.parametrize("n_valid_total", [None, 3 * 150])
def test_fused_linear_cross_entropy_padded_vocab(n_valid_total):
    """GPT-2's vocabulary padded 50257 -> 50304: the padding columns leave the softmax (their dW rows are exactly 0),
    the loss is normalised by ``n_valid_total`` when given, and the token loop runs in chunks with a ragged last
    chunk.  The reference takes the logits from the same GEMM (bf16), so the CE part is held to fp32 bounds.  dh is a
    GEMM of the bf16-rounded d(logits) (2^-9 relative each): 1 ulp + 2^-8 (|dlogits| @ |W|).  dW also rounds its
    running sum to bf16 after each of the three chunks: 1 ulp + 2^-7 (|dlogits|^T @ |h|)."""
    from torchacc_b200.ops.cross_entropy import fused_linear_cross_entropy
    from torchacc_b200.ops.linear import gemm
    gen = torch.Generator(device=DEV).manual_seed(5)
    T, H, V, Vv = 333, 256, 50304, 50257
    h = (torch.randn(T, H, device=DEV, generator=gen) * 0.5).bfloat16().requires_grad_()
    w = (torch.randn(V, H, device=DEV, generator=gen) * 0.2).bfloat16().requires_grad_()
    lab = _labels(T, Vv, gen)
    nvt = None if n_valid_total is None else torch.tensor(float(n_valid_total), device=DEV)
    loss = fused_linear_cross_entropy(h, w, lab, chunk_tokens=128, n_valid_total=nvt, valid_vocab=Vv)
    loss.backward()
    assert bool((w.grad[Vv:] == 0).all()), "padding rows of dW must be exactly 0"
    logits = gemm(h.detach(), w.detach())[:, :Vv]
    nv = float(n_valid_total) if n_valid_total is not None else float((lab != -100).sum())
    rows, lse, g, p, onehot = _ce_ref(logits, lab)
    _check_ce_loss(loss, rows, lse, 1.0 / nv, f"flce loss nvt={n_valid_total}")
    dl = g / nv
    h64, w64 = h.detach().double(), w.detach().double()[:Vv]
    check(h.grad, dl @ w64, f"flce dh nvt={n_valid_total}", floor=2.0 ** -8 * (dl.abs() @ w64.abs()))
    check(w.grad[:Vv], dl.t() @ h64, f"flce dW nvt={n_valid_total}", floor=2.0 ** -7 * (dl.abs().t() @ h64.abs()))


# ---------------------------------------------------------------------------------------------------------------------
# AdamW
# ---------------------------------------------------------------------------------------------------------------------
def _adamw_ref(p, m, v, g, lr, b1, b2, eps, wd, step):
    """fp64 torch.optim.AdamW step from fp32 state, with the hyper-parameters as the kernel receives them (fp32).
    Returns the fp64 (p, m, v) and an absolute error floor for each (derivation inline)."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))        # noqa: E731
    lr, b1, b2, eps, wd = f(lr), f(b1), f(b2), f(eps), f(wd)
    p, m, v, g = p.double(), m.double(), v.double(), g.double()
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    upd = (lr / bc1) * m1 / denom
    pd = p * (1 - lr * wd)
    # m, v: two or three fp32 roundings, each <= 2^-24 of the term it rounds; m's two terms may cancel
    m_mag = (b1 * m).abs() + ((1 - b1) * g).abs()
    floor_m, floor_v = 2.0 ** -21 * m_mag, 2.0 ** -21 * v1.abs()
    # p = p (1 - lr wd) - update: ~8 fp32 roundings in the update (sqrt, 1 / sqrt(bc2), divide, lr / bc1, ...), m's own
    # error carried through (the update of m's magnitude), and the bias corrections: the host computes
    # 1 - powf(b, t) in fp32 (bitwise what earlier versions did), whose absolute error of ~2^-24 is a relative error of
    # 2^-24 / bc, large in the first steps when b2 is close to 1 (1.5e-5 at t = 2, b2 = 0.999)
    upd_mag = (lr / bc1) * m_mag / denom
    floor_p = 2.0 ** -20 * (pd.abs() + upd_mag) + 2.0 ** -23 * (1 / bc1 + 1 / bc2) * upd.abs()
    return (pd - upd, m1, v1), (floor_p, floor_m, floor_v)


def _check_adamw(p, m, v, ref, floors, what):
    for out, r, fl, name in zip((p, m, v), ref, floors, "pmv"):
        check(out, r, f"{what} {name}", ulps=4.0, floor=fl)


def _set_grad(p, g):
    """fp32 gradients go to .grad; bf16 ones to the engine hand-off attribute FusedAdamW reads first."""
    if g.dtype == p.dtype:
        p.grad = g
    else:
        p._tb_grad = g
    return g


def _adamw_param(n, gen, with_lp):
    p = torch.nn.Parameter(torch.randn(n, device=DEV, generator=gen))
    if with_lp:
        p._tb_lp_shard = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    return p


@pytest.mark.parametrize("with_lp", [True, False])
@pytest.mark.parametrize("wd", [0.1, 0.0])
@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 100003, 2 ** 23 + 3])
def test_adamw_matches_fp64(n, grad_dtype, wd, with_lp):
    """200 steps; each is checked against the fp64 step taken from the kernel's own previous fp32 state, so errors do
    not compound and the late bias correction (step 200) is covered.  n = 2^23 + 3 runs the second 16-byte group of
    every trip and the scalar tail; n < 4 is all tail."""
    from torchacc_b200.ops.optim import FusedAdamW
    if (not with_lp or wd == 0.0) and n not in (5, 2 ** 23 + 3):
        pytest.skip("weight decay 0 and no shadow copy: at one small and one large n")
    gen = torch.Generator(device=DEV).manual_seed(n)
    lr, betas, eps = 1e-3, (0.9, 0.999), 1e-8
    p = _adamw_param(n, gen, with_lp)
    opt = FusedAdamW([p], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    steps = 200
    for step in range(1, steps + 1):
        g = _set_grad(p, (torch.randn(n, device=DEV, generator=gen) * (1 + step % 7)).to(grad_dtype))
        st = opt.state[p]
        p0 = p.detach().clone()
        m0 = st["exp_avg"].clone() if st else torch.zeros_like(p0)
        v0 = st["exp_avg_sq"].clone() if st else torch.zeros_like(p0)
        opt.step()
        if step in (1, 2, 3, 10, steps) or step % 37 == 0:
            ref, floors = _adamw_ref(p0, m0, v0, g, lr, betas[0], betas[1], eps, wd, step)
            _check_adamw(p.detach(), st["exp_avg"], st["exp_avg_sq"], ref, floors, f"adamw n={n} step={step}")
            if with_lp:
                assert torch.equal(p._tb_lp_shard, p.detach().bfloat16()), "bf16 shadow is not p.bfloat16()"
    assert opt.state_dict()["state"][0]["step"] == steps


@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [5, 2 ** 23 + 3])
def test_adamw_grad_scale_is_prescaled_gradient(n, grad_dtype):
    """grad_scale multiplies the gradient in fp32: bitwise the same as a step on the pre-scaled fp32 gradient."""
    from torchacc_b200.ops.optim import FusedAdamW
    gen = torch.Generator(device=DEV).manual_seed(11)
    init = torch.randn(n, device=DEV, generator=gen)
    a, b = torch.nn.Parameter(init.clone()), torch.nn.Parameter(init.clone())
    a._tb_lp_shard = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    b._tb_lp_shard = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    oa = FusedAdamW([a], lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1)
    ob = FusedAdamW([b], lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1)
    for step in range(3):
        g = (torch.randn(n, device=DEV, generator=gen) * 100).to(grad_dtype)
        s = torch.tensor([0.37 / (step + 1)], device=DEV)
        _set_grad(a, g)
        oa.grad_scale = s
        oa.step()
        b.grad = g.float() * s
        ob.step()
    for x, y in ((a, b), (oa.state[a]["exp_avg"], ob.state[b]["exp_avg"]),
                 (oa.state[a]["exp_avg_sq"], ob.state[b]["exp_avg_sq"]), (a._tb_lp_shard, b._tb_lp_shard)):
        assert torch.equal(x.detach(), y.detach())


@pytest.mark.parametrize("n", [5, 2 ** 23 + 3])
def test_adamw_found_inf_leaves_state_bitwise(n):
    from torchacc_b200.ops.optim import FusedAdamW
    gen = torch.Generator(device=DEV).manual_seed(3)
    p = _adamw_param(n, gen, True)
    opt = FusedAdamW([p], lr=1e-2)
    p.grad = torch.randn(n, device=DEV, generator=gen)
    opt.step()                                             # non-zero moments
    before = [t.clone() for t in (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], p._tb_lp_shard)]
    opt.found_inf = torch.ones(1, device=DEV)
    p.grad = torch.randn(n, device=DEV, generator=gen)
    opt.step()
    after = (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], p._tb_lp_shard)
    for x, y in zip(before, after):
        assert torch.equal(x, y)


@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
def test_adamw_skipped_steps_do_not_advance_bias_correction(grad_dtype):
    """Three steps skipped for found_inf (the start of fp16 loss scaling), then five real ones: the real steps use the
    bias correction of steps 1..5, as torch's AdamW does, and state_dict() reports step 5.  Counting the skipped
    steps would make the first real update about 0.56x too small (betas 0.9 / 0.95)."""
    from torchacc_b200.ops.optim import FusedAdamW
    gen = torch.Generator(device=DEV).manual_seed(17)
    n = 100003
    lr, betas, eps, wd = 1e-3, (0.9, 0.95), 1e-8, 0.1
    p = _adamw_param(n, gen, True)
    opt = FusedAdamW([p], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    flags = [1, 1, 1, 0, 0, 0, 0, 0]
    taken = 0
    for i, f in enumerate(flags):
        opt.found_inf = torch.tensor([float(f)], device=DEV)
        g = _set_grad(p, torch.randn(n, device=DEV, generator=gen).to(grad_dtype))
        st = opt.state[p]
        p0 = p.detach().clone()
        m0 = st["exp_avg"].clone() if st else torch.zeros_like(p0)
        v0 = st["exp_avg_sq"].clone() if st else torch.zeros_like(p0)
        opt.step()
        if f:
            assert torch.equal(p.detach(), p0)
            continue
        taken += 1
        ref, floors = _adamw_ref(p0, m0, v0, g, lr, betas[0], betas[1], eps, wd, taken)
        _check_adamw(p.detach(), st["exp_avg"], st["exp_avg_sq"], ref, floors, f"adamw after skips, step {taken}")
        assert torch.equal(p._tb_lp_shard, p.detach().bfloat16())
        if i == 5:
            assert opt.state_dict()["state"][0]["step"] == taken      # folding the count mid-run changes nothing
    assert opt.state_dict()["state"][0]["step"] == 5


# ---------------------------------------------------------------------------------------------------------------------
# Gradient norm and scaling
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 1000, 5 * 10 ** 7 + 3])
def test_sqnorm_matches_fp64(n, dtype, ordered):
    """sum((g * pre_scale)^2) over n elements with pre_scale != 1, accumulated onto an existing out[0] by two calls.
    The kernel adds ~190 squares per thread, then trees and block partials in fp32: relative error within 1e-5."""
    from torchacc_b200.ops.optim import _sqnorm
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = (torch.randn(n, device=DEV, generator=gen) * 3).to(dtype)
    g2 = torch.randn(n, device=DEV, generator=gen).to(dtype)
    pre = 0.37
    out = torch.tensor([5.0, 0.0], device=DEV)
    _sqnorm(g, out, pre, ordered=ordered)
    _sqnorm(g2, out, pre, ordered=ordered)
    sq = lambda t: (t.float() * pre).double().square().sum()          # noqa: E731  (the kernel scales in fp32)
    ref = 5.0 + sq(g) + sq(g2)
    rel = abs(float(out[0]) - float(ref)) / float(ref)
    print(f"[ulp] sqnorm n={n} {dtype} ordered={ordered}: relative error {rel:.3g}")
    assert rel <= 1e-5, (float(out[0]), float(ref))
    assert float(out[1]) == 0.0


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_sqnorm_flags_non_finite(dtype, bad, ordered):
    from torchacc_b200.ops.optim import _sqnorm
    n = 3 * 10 ** 6
    g = torch.randn(n, device=DEV).to(dtype)
    g[n - 7] = bad
    out = torch.zeros(2, device=DEV)
    _sqnorm(g, out, 1.0, ordered=ordered)
    assert float(out[1]) == 1.0
    # a finite gradient after a flagged one leaves the flag set
    _sqnorm(torch.ones(10, device=DEV, dtype=dtype), out, 1.0, ordered=ordered)
    assert float(out[1]) == 1.0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 1023, 10 ** 7 + 5])
def test_scale_inplace_bitwise(n, dtype):
    from torchacc_b200.ops.optim import scale_
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = (torch.randn(n, device=DEV, generator=gen) * 1e3).to(dtype)
    s = torch.tensor([0.0123], device=DEV)
    ref = (g.float() * s).to(dtype)
    scale_(g, s)
    assert torch.equal(g, ref)
