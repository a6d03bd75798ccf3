"""MX-FP8 mixture-of-experts experts (``compute.fp8``): the grouped modes of csrc/gemm/gemm_mxfp8.cu bit for bit, the
``_MoEExpertsMXFP8Fn`` op against its PyTorch emulation and against the bf16 experts, and training of the native and
HF MoE models with fp8 experts.

Premise of the exact kernel tests (as ``test_mxfp8_exact`` in test_gemm_kernels_gpu.py): every operand is ``q 2^s``
with |q| <= 8 and s constant over each 32-element scale block, so the quantiser represents it exactly; each scale
block's sum of products is a sum of at most 32 integers of at most 7 bits, which the fp8 datapath holds exactly, and
the scaled block sums stay below 2^24 in units of the tile's smallest power of two (asserted).  So the fp32 result
equals the fp64 reference and the output must equal its single rounding.  The exponents vary per row (A), per expert
(B) and per block, so a wrong expert, scale atom, K block or row shifts a result by a power of two.  The capacity rows
past the device-side tile count hold NaN before quantisation: a GEMM that read them, or their scales, would fail."""
import math

import pytest
import torch

from test_gemm_kernels_gpu import COUNT_PATTERNS, Canvas, _counts, group_layout, mx_operand, verify
from test_gemm_kernels_gpu import BF16, DEV, FP32, TILE_M, _index, _nat, assert_exact_premise, expect_exact

gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
def mx_sorted(counts, offsets, K, gen, row_exp=(-20, 20)):
    """Expert-sorted [capacity, K] bf16 rows of ``mx_operand`` values (per-row exponents in ``row_exp``), zero padding
    rows and two spare tiles of NaN past the last expert.  Returns (x, |q| 2^u per element, per-row exponent)."""
    cap = offsets[-1] + 2 * TILE_M
    x = torch.full((cap, K), float("nan"), dtype=BF16, device=DEV)
    mag = torch.zeros(cap, K, dtype=torch.float64, device=DEV)
    r = torch.zeros(cap, 1, dtype=torch.float64, device=DEV)
    x[:offsets[-1]] = 0
    for e, c in enumerate(counts):
        if c:
            v, m, re = mx_operand(c, K, row_exp, gen)
            s = slice(offsets[e], offsets[e] + c)
            x[s], mag[s], r[s] = v, m, re
    return x, mag, r


def expert_weight(E, rows, cols, gen, along_rows=False):
    """[E*rows, cols] bf16: q 2^(s_e + u), q in [-8, 8], s_e one exponent per expert in [-12, 12], u in [0, 3] per
    32-element block of a row (``along_rows``: per column and 32-row block, the transposed quantisation's blocks)."""
    q = torch.randint(-8, 9, (E * rows, cols), generator=gen, device=DEV).double()
    se = torch.randint(-12, 13, (E, 1, 1), generator=gen, device=DEV).double().expand(E, rows, 1).reshape(E * rows, 1)
    if along_rows:
        u = torch.randint(0, 4, (E * rows // 32, cols), generator=gen, device=DEV).double().repeat_interleave(32, 0)
    else:
        u = torch.randint(0, 4, (E * rows, cols // 32), generator=gen, device=DEV).double().repeat_interleave(32, 1)
    w = (q * torch.exp2(se + u)).to(BF16)
    assert torch.equal(w.double(), q * torch.exp2(se + u))
    return w, q.abs() * torch.exp2(u), se


def _quant(x, row=True, col=False):
    from torchacc_b200.ops import fp8
    return fp8.quantize_mxfp8(x, row, col)


def run_grouped_mx(mode, counts, gen, N, K, num_sms=None):
    """mode fwd: D = A B_e^T with B [E*N, K]; dgrad: B_e^T from the transposed quantisation of W [E*K, N]."""
    from torchacc_b200.ops import fp8
    nat, L = _nat()
    E = len(counts)
    offsets, tile_expert = group_layout(counts)
    te, nmt, _ = _index(counts, offsets, tile_expert)
    a, amag, ra = mx_sorted(counts, offsets, K, gen)
    cap, valid = a.shape[0], offsets[-1]
    ar, _ = _quant(a)
    if mode == "fwd":
        w, wmag, se = expert_weight(E, N, K, gen)
        br, _ = _quant(w)
        bq = br
        b_deq = fp8.dequantize_mxfp8(br).double()                     # [E*N, K]
    else:
        w, wmag, se = expert_weight(E, K, N, gen, along_rows=True)    # [E*K, N]
        _, bq = _quant(w, False, True)                                 # [N, E*K]
        b_deq = fp8.dequantize_mxfp8(bq).double()
    assert torch.equal(fp8.dequantize_mxfp8(ar)[:valid].double(), a[:valid].double()), "quantiser not exact"
    assert torch.equal(b_deq, w.double() if mode == "fwd" else w.double().t()), "quantiser not exact"
    d = Canvas(cap, N, BF16)
    nat.check(L.tb_gemm_grouped_mxfp8(ar.q.data_ptr(), ar.sf.data_ptr(), bq.q.data_ptr(), bq.sf.data_ptr(),
                                      d.view.data_ptr(), cap, N, K, E, ar.q.stride(0), bq.q.stride(0), d.pitch,
                                      int(mode == "dgrad"), te.data_ptr(), nmt.data_ptr(), num_sms or nat.num_sms(),
                                      nat.stream()), "tb_gemm_grouped_mxfp8")
    torch.cuda.synchronize()
    ref = torch.zeros(valid, N, dtype=torch.float64, device=DEV)
    for e in range(E):
        r = slice(offsets[e], offsets[e + 1])
        if r.stop == r.start:
            continue
        be = b_deq[e * N:(e + 1) * N] if mode == "fwd" else b_deq[:, e * K:(e + 1) * K]
        bm = wmag[e * N:(e + 1) * N] if mode == "fwd" else wmag[e * K:(e + 1) * K].t()
        assert_exact_premise((amag[r] @ bm.t()).max(), f"grouped mxfp8 {mode}")
        ref[r] = a[r].double() @ be.t()
    expect_exact(d.view[:valid], ref, f"grouped mxfp8 {mode} E={E}")
    pad = torch.ones(valid, dtype=torch.bool, device=DEV)
    for e, c in enumerate(counts):
        pad[offsets[e]:offsets[e] + c] = False
    assert bool((d.view[:valid][pad] == 0).all()), "padding rows must be exact zeros"
    d.check_untouched(f"grouped mxfp8 {mode}: rows past the device-side tile count", written_rows=valid)
    print(f"[exact] grouped mxfp8 {mode} E={E} N={N} K={K} sms={num_sms}: {valid} rows exact, spare tiles untouched")


def run_grouped_wgrad_mx(out, counts, gen, M, N, num_sms=None):
    """D_e [M, N] (+)= dY_e^T X_e from the transposed quantisations; out: fp32, bf16, fp32_acc, bf16_acc.  Both operands
    are q 2^(s_e + u_b + u_c): one exponent per expert, one per 32-token block (the scale blocks of the transposed
    quantisation, so a wrong K block or scale atom inside an expert changes the result) and one per column (so does a
    wrong row atom of A or B)."""
    from torchacc_b200.ops import fp8
    nat, L = _nat()
    E = len(counts)
    offsets, _ = group_layout(counts)
    _, _, off = _index(counts, offsets, [])
    cap = offsets[-1] + 2 * TILE_M
    valid = offsets[-1]

    def operand(C):
        q = torch.randint(-8, 9, (cap, C), generator=gen, device=DEV).double()
        s = torch.zeros(cap, 1, dtype=torch.float64, device=DEV)
        for e in range(E):
            s[offsets[e]:offsets[e + 1]] = float(torch.randint(-10, 11, (1,), generator=gen, device=DEV))
        u = (torch.randint(0, 3, (cap // 32, 1), generator=gen, device=DEV).double().repeat_interleave(32, 0)
             + torch.randint(0, 2, (1, C), generator=gen, device=DEV).double())
        v = q * torch.exp2(s + u)
        for e, c in enumerate(counts):
            v[offsets[e] + c:offsets[e + 1]] = 0                     # padding rows
        v[valid:] = float("nan")                                     # capacity past the device-side tile count
        return v.to(BF16), q.abs() * torch.exp2(u), s

    dy, dmag, ds = operand(M)
    x, xmag, xs = operand(N)
    _, dyc = _quant(dy, False, True)
    _, xc = _quant(x, False, True)
    assert torch.equal(fp8.dequantize_mxfp8(dyc)[:, :valid].double(), dy[:valid].double().t())
    assert torch.equal(fp8.dequantize_mxfp8(xc)[:, :valid].double(), x[:valid].double().t())
    out_dtype = FP32 if out.startswith("fp32") else BF16
    acc = out.endswith("acc")
    ref = torch.zeros(E * M, N, dtype=torch.float64, device=DEV)
    init = None
    if acc:
        init = torch.randint(-2000, 2001, (E * M, N), generator=gen, device=DEV).double()
    for e in range(E):
        r = slice(offsets[e], offsets[e + 1])
        grid = torch.exp2(ds[offsets[e]] + xs[offsets[e]]) if r.stop > r.start else torch.ones(1, device=DEV).double()
        if init is not None:
            init[e * M:(e + 1) * M] *= grid
        if r.stop > r.start:
            assert_exact_premise((dmag[r].t() @ xmag[r]).max() + 2000, "grouped mxfp8 wgrad")
            ref[e * M:(e + 1) * M] = dy[r].double().t() @ x[r].double()
    if init is not None:
        init = init.to(out_dtype)
        ref += init.double()
    d = Canvas(E * M, N, out_dtype, init=init, gap=24)
    nat.check(L.tb_gemm_grouped_wgrad_mxfp8(dyc.q.data_ptr(), dyc.sf.data_ptr(), xc.q.data_ptr(), xc.sf.data_ptr(),
                                            d.view.data_ptr(), M, N, E, cap, dyc.q.stride(0), xc.q.stride(0), d.pitch,
                                            off.data_ptr(), int(out_dtype == FP32), int(acc),
                                            num_sms or nat.num_sms(), nat.stream()), "tb_gemm_grouped_wgrad_mxfp8")
    torch.cuda.synchronize()
    verify(d, ref, f"grouped mxfp8 wgrad {out} E={E} M={M} N={N} sms={num_sms}")


@gpu
@pytest.mark.parametrize("pattern", list(COUNT_PATTERNS))
@pytest.mark.parametrize("mode", ["fwd", "dgrad"])
def test_grouped_mxfp8_exact(mode, pattern):
    """Experts with 0, 1, 127, 128, 129 rows, one expert taking every row, 128 experts.  Forward N = 256 (B_e's rows
    must start on a scale atom); dgrad N = 200, a tail of the 128-wide output tile.  K = 384, three K blocks."""
    gen = torch.Generator(device=DEV).manual_seed(31)
    counts = _counts(pattern, gen)
    run_grouped_mx(mode, counts, gen, N=256 if mode == "fwd" else 200, K=384)


@gpu
@pytest.mark.parametrize("pattern", list(COUNT_PATTERNS))
@pytest.mark.parametrize("out", ["fp32", "bf16", "fp32_acc", "bf16_acc"])
def test_grouped_wgrad_mxfp8_exact(out, pattern):
    """Empty experts are zeroed, or left unchanged when accumulating; M = 200 and N = 136 are tile tails; D is a view
    with a pitch gap."""
    gen = torch.Generator(device=DEV).manual_seed(32)
    run_grouped_wgrad_mx(out, _counts(pattern, gen), gen, M=200, N=136)


@gpu
@pytest.mark.parametrize("mode", ["fwd", "dgrad", "wgrad"])
def test_grouped_mxfp8_persistent_loop(mode):
    """1, 2 and 3 CTAs for the whole grouped problem: many tiles (wgrad: many experts' K ranges) per CTA."""
    gen = torch.Generator(device=DEV).manual_seed(33)
    counts = [129, 0, 300, 1, 128, 0, 640, 5]
    for sms in (1, 2, 3):
        if mode == "wgrad":
            run_grouped_wgrad_mx("fp32_acc" if sms != 2 else "bf16", counts, gen, M=200, N=296, num_sms=sms)
        else:
            run_grouped_mx(mode, counts, gen, N=384 if mode == "fwd" else 520, K=256, num_sms=sms)


@gpu
def test_grouped_mxfp8_qwen3_moe_shape():
    """Qwen3-30B-A3B: 128 experts, top-8 routing of 2048 tokens, H = 2048, F = 768: gate|up (N = 2F, K = H), down
    (N = H, K = F), down dgrad (N = F, K = H) and down wgrad (M = H, N = F) into fp32."""
    gen = torch.Generator(device=DEV).manual_seed(34)
    E, k, T, H, F = 128, 8, 2048, 2048, 768
    ids = torch.rand(T, E, generator=torch.Generator().manual_seed(3)).topk(k, dim=1).indices
    counts = torch.bincount(ids.reshape(-1), minlength=E).tolist()
    run_grouped_mx("fwd", counts, gen, N=2 * F, K=H)
    run_grouped_mx("fwd", counts, gen, N=H, K=F)
    run_grouped_mx("dgrad", counts, gen, N=F, K=H)
    run_grouped_wgrad_mx("fp32", counts, gen, M=H, N=F)


@gpu
def test_grouped_mxfp8_rejects_bad_shapes():
    """K % 128 != 0, a forward N that splits a scale atom between experts and misaligned pitches are refused."""
    nat, L = _nat()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    te = torch.zeros(4, dtype=torch.int32, device=DEV)
    p = buf.data_ptr()
    args = lambda N, K, lda, bt: (p, p, p, p, p, 256, N, K, 2, lda, K, N, bt, te.data_ptr(), te.data_ptr(), 1,
                                  nat.stream())
    assert L.tb_gemm_grouped_mxfp8(*args(256, 192, 192, 0)) != 0        # K % 128
    assert L.tb_gemm_grouped_mxfp8(*args(200, 256, 256, 0)) != 0        # forward N % 128
    assert L.tb_gemm_grouped_mxfp8(*args(256, 256, 264, 0)) != 0        # lda % 16
    assert L.tb_gemm_grouped_wgrad_mxfp8(p, p, p, p, p, 128, 128, 2, 192, 192, 192, 128, te.data_ptr(), 1, 0, 1,
                                         nat.stream()) != 0             # rows % 128
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the op
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def fp8_on():
    from torchacc_b200.ops import fp8
    prev = fp8.enabled()
    fp8.enable(True)
    yield
    fp8.enable(prev)


def _case(T=512, H=256, Fd=384, E=8, k=2, seed=3, dtype=BF16):
    torch.manual_seed(seed)
    x = torch.randn(T, H, device=DEV, dtype=dtype)
    logits = torch.randn(T, E, device=DEV)
    w, ids = torch.topk(torch.softmax(logits, -1), k, -1)
    w = w / w.sum(-1, keepdim=True)
    wgu = (torch.randn(E, 2 * Fd, H, device=DEV) / math.sqrt(H)).to(dtype)
    wd = (torch.randn(E, H, Fd, device=DEV) / math.sqrt(Fd)).to(dtype)
    return x, ids, w, wgu, wd


def _run(x, ids, w, wgu, wd, dout, residual=None):
    from torchacc_b200.ops.moe import moe_experts
    leaves = [t.clone().requires_grad_(True) for t in (x, w, wgu, wd)]
    out = moe_experts(leaves[0], ids, leaves[1], leaves[2], leaves[3], residual=residual)
    out.backward(dout)
    return [out.detach()] + [t.grad for t in leaves]


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


NAMES = ("out", "dx", "dweights", "dW_gate_up", "dW_down")


@gpu
@pytest.mark.parametrize("shape", [dict(), dict(T=1000, H=384, Fd=256, E=16, k=4), dict(T=300, E=128, k=8, Fd=128)],
                         ids=["mixtral_like", "e16k4", "e128k8"])
def test_fp8_experts_match_emulation(shape, fp8_on):
    """Native MX-FP8 experts against ``moe_experts_mxfp8_reference``, which quantises the same operands the same way
    and rounds to bf16 at the same points.  What remains is the fp32 accumulation order (below 2^-20 of a result) and
    the fp32 sigmoid of the SwiGLU kernel (a few fp32 ulps).  Either can flip a bf16 rounding of an intermediate (one
    bf16 ulp, 2^-8 relative) and that element's e4m3 rounding (one e4m3 ulp, 2^-3 relative of that one element) in the
    next GEMM.  Flips are rare (they need a value within a few fp32 ulps of a rounding boundary), and each touches one
    of the >= 128 terms of a contraction, so a relative Frobenius error of 2^-7 leaves a wide margin over every
    output."""
    from torchacc_b200.ops import moe as moe_mod
    x, ids, w, wgu, wd = _case(**shape)
    dout = torch.randn_like(x)
    calls = moe_mod.FP8_EXPERT_CALLS
    got = _run(x, ids, w, wgu, wd, dout)
    assert moe_mod.FP8_EXPERT_CALLS == calls + 1
    ref = moe_mod.moe_experts_mxfp8_reference(x, ids, w, wgu, wd, dout=dout)
    bound = 2.0 ** -7
    for name, a, b in zip(NAMES, got, ref):
        assert torch.isfinite(a).all(), name
        rel = _rel(a, b)
        print(f"[bound] fp8 experts vs emulation {name}: rel {rel:.3g}, {rel / bound:.3f} of the bound")
        assert rel < bound, (name, rel)


@gpu
def test_fp8_experts_close_to_bf16(fp8_on):
    """Close to the bf16 native experts.  ``test_fp8_linear_fwd_bwd_close_to_bf16`` bounds one fp8 GEMM (two quantised
    operands, about 0.027 relative error each on Gaussian data) by a relative norm of 0.06.  Every expert output and
    gradient here goes through two chained fp8 GEMMs whose quantisation errors are independent, so they add in
    quadrature: sqrt(2) * 0.06 = 0.085.  (The fp64 emulation on the CPU gives 0.066-0.069 at several shapes.)"""
    from torchacc_b200.ops import fp8
    x, ids, w, wgu, wd = _case(T=1024, H=512, Fd=512, E=8, k=2)
    dout = torch.randn_like(x)
    got = _run(x, ids, w, wgu, wd, dout)
    fp8.enable(False)
    ref = _run(x, ids, w, wgu, wd, dout)
    for name, a, b in zip(NAMES, got, ref):
        rel = _rel(a, b)
        print(f"[bound] fp8 vs bf16 experts {name}: rel {rel:.4f} (bound 0.085)")
        assert rel < 0.085, (name, rel)


@gpu
def test_fp8_experts_bitwise_repeatable_and_sentinels(fp8_on):
    """Two runs are bitwise equal.  Ids equal to E (HF's "no expert") add nothing and get a zero weight gradient."""
    from torchacc_b200.ops import moe as moe_mod
    x, ids, w, wgu, wd = _case(T=512, E=8, k=2)
    ids = ids.clone()
    ids[::7, 1] = 8
    dout = torch.randn_like(x)
    a = _run(x, ids, w, wgu, wd, dout)
    b = _run(x, ids, w, wgu, wd, dout)
    for name, u, v in zip(NAMES, a, b):
        assert torch.equal(u, v), name
    assert bool((a[2][::7, 1] == 0).all()), "a sentinel id got a non-zero weight gradient"
    ref = moe_mod.moe_experts_mxfp8_reference(x, ids, w, wgu, wd, dout=dout)
    for name, u, v in zip(NAMES, a, ref):
        assert _rel(u, v) < 2.0 ** -7, name


@gpu
def test_fp8_experts_hold_nothing_under_checkpointing(fp8_on):
    """Under non-reentrant activation checkpointing (what ``memory.gc`` uses) the experts keep nothing of their own
    between the forward and the backward: the fp8 activation copies go through ``save_for_backward``, so the
    checkpoint drops them and its recompute regenerates them, and the fp8 weight copies never outlive a pass.  The
    memory that stays allocated after the fp8 forward is the output alone (the bf16 experts hold no less), and the
    checkpointed fp8 run computes bitwise what the plain one does."""
    from torch.utils.checkpoint import checkpoint
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops import moe as moe_mod
    x, ids, w, wgu, wd = _case(T=2048, H=512, Fd=512, E=8, k=2)
    dout = torch.randn_like(x)

    def run(on):
        fp8.enable(on)
        calls = moe_mod.FP8_EXPERT_CALLS
        leaves = [t.clone().requires_grad_(True) for t in (x, w, wgu, wd)]
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        out = checkpoint(moe_mod.moe_experts, leaves[0], ids, leaves[1], leaves[2], leaves[3], use_reentrant=False)
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - before
        out.backward(dout)
        assert moe_mod.FP8_EXPERT_CALLS - calls == (2 if on else 0)       # forward and recompute
        return held, out.numel() * out.element_size(), [out.detach()] + [t.grad for t in leaves]

    held, out_bytes, got = run(True)
    held_bf16, _, _ = run(False)
    print(f"[memory] held after a checkpointed forward: fp8 {held} B, bf16 {held_bf16} B, output {out_bytes} B")
    assert held == out_bytes and held <= held_bf16, (held, held_bf16, out_bytes)
    fp8.enable(True)
    plain = _run(x, ids, w, wgu, wd, dout)
    for name, a, b in zip(NAMES, got, plain):
        assert torch.equal(a, b), name


@gpu
def test_fp8_experts_no_host_sync(fp8_on):
    from torchacc_b200.ops import moe as moe_mod
    from torchacc_b200.ops.moe import moe_experts, moe_router
    x, ids, w, wgu, wd = _case()
    logits = torch.randn(x.shape[0], 8, device=DEV, dtype=BF16, requires_grad=True)
    leaves = [t.clone().requires_grad_(True) for t in (x, wgu, wd)]
    wr, idr = moe_router(logits, 2, True)
    moe_experts(leaves[0], idr, wr, leaves[1], leaves[2]).float().sum().backward()   # warm-up
    calls = moe_mod.FP8_EXPERT_CALLS
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        wr, idr = moe_router(logits, 2, True)
        out = moe_experts(leaves[0], idr, wr, leaves[1], leaves[2])
        out.float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert moe_mod.FP8_EXPERT_CALLS == calls + 1
    assert logits.grad is not None and leaves[1].grad is not None and leaves[2].grad is not None


@gpu
def test_fp8_off_and_ineligible_take_the_bf16_path():
    """fp8 off: outputs bitwise equal to the bf16 experts.  A hidden size that is not a multiple of 128 (the native
    experts already need F % 128 == 0), and fp16, keep the 16-bit experts with fp8 on: the counter does not move and the
    results are bitwise those of the 16-bit path."""
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops import moe as moe_mod
    prev = fp8.enabled()
    try:
        cases = [(dict(), False), (dict(H=200), True), (dict(dtype=torch.float16), True)]
        for shape, on in cases:
            x, ids, w, wgu, wd = _case(**shape)
            dout = torch.randn_like(x)
            fp8.enable(False)
            leaves = [t.clone().requires_grad_(True) for t in (x, w, wgu, wd)]
            ref_out = moe_mod._MoEExpertsFn.apply(leaves[0], leaves[1], leaves[2], leaves[3], ids, None, None)
            ref_out.backward(dout)
            ref = [ref_out.detach()] + [t.grad for t in leaves]
            fp8.enable(on)
            calls = moe_mod.FP8_EXPERT_CALLS
            got = _run(x, ids, w, wgu, wd, dout)
            assert moe_mod.FP8_EXPERT_CALLS == calls, shape
            for name, a, b in zip(NAMES, got, ref):
                assert torch.equal(a, b), (shape, name)
    finally:
        fp8.enable(prev)


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _train(preset, use_fp8, steps=4, seed=0):
    import torchacc_b200 as ta
    from torchacc_b200.models import build_llama
    from torchacc_b200.ops import moe as moe_mod
    torch.manual_seed(seed)
    with torch.device(DEV):
        model = build_llama(preset, dtype=torch.bfloat16)
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.compute.fp8 = use_fp8
    cfg.compute.deterministic = True
    cfg.memory.gc = True
    cfg.memory.gc_cls = {"LlamaDecoderLayer"}
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=3e-3)
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(0, 512, (2, 256), device=DEV, generator=g)
    calls = moe_mod.FP8_EXPERT_CALLS
    losses = []
    try:
        for _ in range(steps):
            out = model(input_ids=ids, labels=ids)
            out["loss"].backward()
            model.clip_grad_norm_(1.0)
            opt.step()
            model.zero_grad()
            losses.append(out["loss"].detach().clone())
    finally:
        from torchacc_b200.ops import fp8
        fp8.enable(False)
    params = [p.detach().clone() for p in model.parameters()]
    return losses, params, moe_mod.FP8_EXPERT_CALLS - calls, model.engine.stats.get("wgrad_fallbacks", 0)


@gpu
@pytest.mark.parametrize("preset", ["tiny-moe", "tiny-qwen3-moe"])
def test_native_moe_training_with_fp8_experts(preset):
    """FSDP + activation checkpointing with ``compute.fp8``: the experts run in fp8 (forward and checkpoint recompute of
    both layers every step), every expert weight gradient lands in the flat buffer, two runs are bitwise equal and the
    loss decreases.  Against the bf16 run: the first loss (identical weights) within 0.01, where the experts' ~7 %
    relative output error moves a ~6.2 loss by about 1e-3; the later losses within 0.25, since Adam at lr 3e-3 turns
    the ~7 % gradient difference into different updates and the two runs drift apart step by step (0.13 and 0.05
    after four steps on an H100)."""
    l1, p1, calls, fallbacks = _train(preset, True)
    assert calls >= 4 * 2, f"fp8 experts ran {calls} times"
    assert fallbacks == 0
    l2, p2, _, _ = _train(preset, True)
    for a, b in zip(l1, l2):
        assert torch.equal(a, b)
    for a, b in zip(p1, p2):
        assert torch.equal(a, b)
    assert float(l1[-1]) < float(l1[0]), [float(v) for v in l1]
    lb, _, calls_bf16, _ = _train(preset, False)
    assert calls_bf16 == 0
    diffs = [abs(float(a) - float(b)) for a, b in zip(l1, lb)]
    print(f"[bound] {preset} losses fp8 {[float(v) for v in l1]} bf16 {[float(v) for v in lb]}")
    assert diffs[0] < 0.01, diffs
    assert max(diffs) < 0.25, diffs


@gpu
def test_hf_mixtral_fp8_experts_close_to_bf16():
    """A tiny HF Mixtral through ``accelerate`` with fixed routing: fp8 experts against the bf16 run of the same model,
    loss within 0.03 and every gradient (per flat-buffer unit) within a relative norm of 0.1."""
    import copy
    transformers = pytest.importorskip("transformers")
    import torchacc_b200 as ta
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops import moe as moe_mod
    from test_moe_gpu import _fix_routing
    torch.manual_seed(0)
    cfg = transformers.MixtralConfig(vocab_size=256, hidden_size=256, intermediate_size=256, num_hidden_layers=2,
                                     num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                                     max_position_embeddings=256, num_local_experts=8, num_experts_per_tok=2,
                                     tie_word_embeddings=False, router_aux_loss_coef=0.0)
    base = transformers.MixtralForCausalLM(cfg).to(DEV, torch.bfloat16)
    g = torch.Generator(device=DEV).manual_seed(3)
    ids = torch.randint(0, 256, (2, 128), device=DEV, generator=g)
    table = [torch.rand(256, 8, device=DEV, generator=g).argsort(-1)[:, :2] for _ in range(2)]
    results = []
    try:
        for use_fp8 in (False, True):
            model = copy.deepcopy(base)
            _fix_routing(model, table)
            tcfg = ta.Config()
            tcfg.compute.bf16 = True
            tcfg.compute.fp8 = use_fp8
            model = ta.accelerate(model, config=tcfg)
            calls = moe_mod.FP8_EXPERT_CALLS
            out = model(input_ids=ids, labels=ids)
            out["loss"].backward()
            assert moe_mod.FP8_EXPERT_CALLS - calls == (2 if use_fp8 else 0)
            eng = model.engine
            grads = eng.grads() if eng is not None else [p.grad for p in model.parameters() if p.grad is not None]
            results.append((float(out["loss"]), [t.float().clone() for t in grads]))
    finally:
        fp8.enable(False)
    (lb, gb), (lf, gf) = results
    assert abs(lf - lb) < 0.03, (lf, lb)
    assert len(gb) == len(gf) and gb
    for i, (a, b) in enumerate(zip(gf, gb)):
        rel = float((a - b).norm() / b.norm().clamp(min=1e-30))
        print(f"[bound] HF Mixtral fp8 vs bf16 gradient {i}: rel {rel:.4f} (bound 0.1)")
        assert rel < 0.1, (i, rel)
