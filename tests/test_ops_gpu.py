"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _close(a, b, rtol, atol, what=""):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}, max ref {b.abs().max().item():.4g}"


@pytest.mark.parametrize("M,N,K", [(256, 512, 128), (1000, 776, 328), (4096, 4096, 1024), (77, 136, 72)])
@pytest.mark.parametrize("bias", [False, True])
def test_linear_fwd_bwd(M, N, K, bias):
    from torchacc_b200.ops.linear import linear
    from torchacc_b200 import _native as nat
    assert nat.available()
    torch.manual_seed(0)
    x = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16().requires_grad_()
    w = (torch.randn(N, K, device=_dev()) * 0.1).bfloat16().requires_grad_()
    b = (torch.randn(N, device=_dev())).bfloat16().requires_grad_() if bias else None
    n0 = nat.LAUNCHES
    y = linear(x, w, b)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert nat.LAUNCHES - n0 >= 3, "native GEMM was not used"
    xf, wf = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    bf = b.detach().float().requires_grad_() if bias else None
    yr = F.linear(xf, wf, bf)
    yr.backward(dy.float())
    _close(y, yr, 1e-2, 1e-2 * math.sqrt(K) * 0.05 + 1e-2, "y")
    _close(x.grad, xf.grad, 2e-2, 2e-2 * math.sqrt(N) * 0.1 + 1e-2, "dx")
    _close(w.grad, wf.grad, 2e-2, 2e-2 * math.sqrt(M) * 0.5 + 1e-2, "dw")
    if bias:
        _close(b.grad, bf.grad, 2e-2, 0.5, "db")


def test_gemm_accumulate_into_view():
    from torchacc_b200.ops.linear import gemm
    torch.manual_seed(1)
    a = torch.randn(512, 256, device=_dev()).bfloat16()
    b = torch.randn(384, 256, device=_dev()).bfloat16()
    flat = torch.zeros(384 * 512 + 64, device=_dev(), dtype=torch.bfloat16)
    view = flat[64:].view(512, 384)
    gemm(a, b, out=view)
    gemm(a, b, out=view, accumulate=True)
    ref = 2 * (a.float() @ b.float().t())
    _close(view, ref, 2e-2, 0.5, "accumulate")
    out32 = torch.zeros(512, 384, device=_dev(), dtype=torch.float32)
    gemm(a, b, out=out32)
    _close(out32, ref / 2, 1e-3, 1e-2, "fp32 out")


@pytest.mark.parametrize("shape", [(512, 384, 256), (200, 328, 136)])
def test_linear_with_fused_residual(shape):
    """y = x W^T + b + residual in ONE GEMM (epilogue addend); gradients of x, W, b and of the residual branch."""
    from torchacc_b200.ops.linear import gemm, linear
    M, N, K = shape
    torch.manual_seed(2)
    x = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16().requires_grad_()
    w = (torch.randn(N, K, device=_dev()) * 0.1).bfloat16().requires_grad_()
    b = torch.randn(N, device=_dev()).bfloat16().requires_grad_()
    r = torch.randn(M, N, device=_dev()).bfloat16().requires_grad_()
    y = linear(x, w, b, residual=r)
    dy = torch.randn_like(y)
    y.backward(dy)
    xf, wf, bf, rf = (t.detach().float().requires_grad_() for t in (x, w, b, r))
    yr = F.linear(xf, wf, bf) + rf
    yr.backward(dy.float())
    _close(y, yr, 2e-2, 5e-2, "y")
    _close(x.grad, xf.grad, 2e-2, 5e-2, "dx")
    _close(w.grad, wf.grad, 2e-2, 0.3, "dw")
    _close(r.grad, rf.grad, 0, 0, "dresidual")
    # fp32 output with an fp32 addend that is not the output buffer
    c32 = torch.randn(M, N, device=_dev())
    o32 = gemm(x.detach(), w.detach(), out_dtype=torch.float32, addend=c32)
    _close(o32, x.detach().float() @ w.detach().float().t() + c32, 1e-3, 1e-2, "fp32 addend")


def test_rmsnorm_passthrough_sums_skip_gradient():
    """rmsnorm(..., passthrough=True) hands the input back as a second output; the gradient arriving on it is added
    to dx inside the backward kernel (no separate accumulation pass)."""
    from torchacc_b200.ops.rmsnorm import rmsnorm
    torch.manual_seed(3)
    T, H = 257, 4096
    x = torch.randn(T, H, device=_dev()).bfloat16().requires_grad_()
    w = (1 + 0.1 * torch.randn(H, device=_dev())).bfloat16().requires_grad_()
    y, skip = rmsnorm(x, w, 1e-5, passthrough=True)
    assert skip.data_ptr() == x.data_ptr()
    dy, ds = torch.randn_like(y), torch.randn_like(y)
    torch.autograd.backward([y, skip], [dy, ds])
    xf, wf = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    yr = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    torch.autograd.backward([yr, xf * 1.0], [dy.float(), ds.float()])
    _close(x.grad, xf.grad, 3e-2, 3e-2, "dx")
    _close(w.grad, wf.grad, 3e-2, 0.3, "dw")


@pytest.mark.parametrize("H", [256, 4096, 8192, 1000 * 8])
@pytest.mark.parametrize("residual", [False, True])
def test_rmsnorm(H, residual):
    from torchacc_b200.ops.rmsnorm import rmsnorm, rmsnorm_ref
    torch.manual_seed(0)
    T = 333
    x = torch.randn(T, H, device=_dev()).bfloat16().requires_grad_()
    r = torch.randn(T, H, device=_dev()).bfloat16().requires_grad_() if residual else None
    w = (1 + 0.1 * torch.randn(H, device=_dev())).bfloat16().requires_grad_()
    y, h = rmsnorm(x, w, 1e-5, r)
    dy = torch.randn_like(y)
    dh = torch.randn_like(y) if residual else None
    if residual:
        torch.autograd.backward([y, h], [dy, dh])
    else:
        y.backward(dy)
    xf = x.detach().float().requires_grad_()
    rf = r.detach().float().requires_grad_() if residual else None
    wf = w.detach().float().requires_grad_()
    hf = xf + rf if residual else xf
    if residual:
        hf = hf.bfloat16().float()  # the residual stream is stored in bf16 (the cast is differentiable)
    yr = hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    if residual:
        torch.autograd.backward([yr, hf], [dy.float(), dh.float()])
    else:
        yr.backward(dy.float())
    _close(y, yr, 2e-2, 2e-2, "y")
    _close(x.grad, xf.grad, 3e-2, 3e-2, "dx")
    _close(w.grad, wf.grad, 3e-2, 0.3, "dw")
    if residual:
        _close(r.grad, rf.grad, 3e-2, 3e-2, "dres")


def test_rope_qkv_inplace_matches_reference():
    from torchacc_b200.ops.rope import rope_qkv_, rope_tables, _rope_ref
    torch.manual_seed(0)
    B, S, hq, hk, D = 2, 96, 8, 2, 128
    T = B * S
    cos, sin = rope_tables(256, D, 500000.0, _dev())
    qkv0 = torch.randn(T, (hq + 2 * hk) * D, device=_dev()).bfloat16()
    src = qkv0.clone().requires_grad_()
    qkv = rope_qkv_(src * 1.0, hq, hk, D, cos, sin, None, S)
    pos = torch.arange(T, device=_dev()) % S
    q_ref = _rope_ref(qkv0[:, :hq * D].reshape(T, hq, D), cos, sin, pos, 1.0)
    k_ref = _rope_ref(qkv0[:, hq * D:(hq + hk) * D].reshape(T, hk, D), cos, sin, pos, 1.0)
    _close(qkv[:, :hq * D].reshape(T, hq, D), q_ref, 1e-2, 1e-2, "q")
    _close(qkv[:, hq * D:(hq + hk) * D].reshape(T, hk, D), k_ref, 1e-2, 1e-2, "k")
    assert torch.equal(qkv[:, (hq + hk) * D:], qkv0[:, (hq + hk) * D:])
    g = torch.randn_like(qkv)
    qkv.backward(g)
    gq = _rope_ref(g[:, :hq * D].reshape(T, hq, D), cos, sin, pos, -1.0)
    _close(src.grad[:, :hq * D].reshape(T, hq, D), gq, 1e-2, 1e-2, "dq")
    assert torch.equal(src.grad[:, (hq + hk) * D:], g[:, (hq + hk) * D:])
    # explicit positions
    p = torch.randint(0, 200, (T,), device=_dev(), dtype=torch.int32)
    q2 = rope_qkv_(qkv0.clone(), hq, hk, D, cos, sin, p, S)
    _close(q2[:, :hq * D].reshape(T, hq, D), _rope_ref(qkv0[:, :hq * D].reshape(T, hq, D), cos, sin, p, 1.0), 1e-2, 1e-2)


def test_swiglu():
    from torchacc_b200.ops.swiglu import swiglu, swiglu_separate
    torch.manual_seed(0)
    T, Fd = 300, 1408
    gu = torch.randn(T, 2 * Fd, device=_dev()).bfloat16().requires_grad_()
    h = swiglu(gu)
    dh = torch.randn_like(h)
    h.backward(dh)
    guf = gu.detach().float().requires_grad_()
    hr = F.silu(guf[:, :Fd]) * guf[:, Fd:]
    hr.backward(dh.float())
    _close(h, hr, 1e-2, 1e-2, "h")
    _close(gu.grad, guf.grad, 2e-2, 2e-2, "dgu")
    g = torch.randn(T, Fd, device=_dev()).bfloat16().requires_grad_()
    u = torch.randn(T, Fd, device=_dev()).bfloat16().requires_grad_()
    h2 = swiglu_separate(g, u)
    h2.backward(dh)
    gf, uf = g.detach().float().requires_grad_(), u.detach().float().requires_grad_()
    (F.silu(gf) * uf).backward(dh.float())
    _close(g.grad, gf.grad, 2e-2, 2e-2, "dg")
    _close(u.grad, uf.grad, 2e-2, 2e-2, "du")


@pytest.mark.parametrize("V", [1024, 128256, 50264])
def test_cross_entropy(V):
    from torchacc_b200.ops.cross_entropy import cross_entropy
    torch.manual_seed(0)
    n = 64
    logits = (torch.randn(n, V, device=_dev()) * 2).bfloat16().requires_grad_()
    labels = torch.randint(0, V, (n,), device=_dev())
    labels[::7] = -100
    loss = cross_entropy(logits, labels)
    loss.backward()
    lf = logits.detach().float().requires_grad_()
    lr = F.cross_entropy(lf, labels, ignore_index=-100)
    lr.backward()
    assert abs(float(loss) - float(lr)) < 2e-3 * max(1.0, abs(float(lr)))
    _close(logits.grad, lf.grad, 2e-2, 2e-4, "dlogits")


def test_fused_linear_cross_entropy():
    from torchacc_b200.ops.cross_entropy import fused_linear_cross_entropy
    torch.manual_seed(0)
    T, H, V = 700, 512, 4096
    h = torch.randn(T, H, device=_dev()).bfloat16().requires_grad_()
    w = (torch.randn(V, H, device=_dev()) * 0.05).bfloat16().requires_grad_()
    labels = torch.randint(0, V, (T,), device=_dev())
    labels[:50] = -100
    loss = fused_linear_cross_entropy(h, w, labels, chunk_tokens=256)
    loss.backward()
    hf, wf = h.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    lr = F.cross_entropy(F.linear(hf, wf), labels, ignore_index=-100)
    lr.backward()
    assert abs(float(loss) - float(lr)) < 5e-3 * max(1.0, abs(float(lr))), (float(loss), float(lr))
    _close(h.grad, hf.grad, 5e-2, 5e-5, "dh")
    _close(w.grad, wf.grad, 5e-2, 5e-5, "dw")


@pytest.mark.parametrize("gdtype", [torch.bfloat16, torch.float32])
def test_fused_adamw_matches_torch(gdtype):
    from torchacc_b200.ops.optim import FusedAdamW
    torch.manual_seed(0)
    n = 100003
    p0 = torch.randn(n, device=_dev())
    p = torch.nn.Parameter(p0.clone())
    lp = torch.zeros(n, device=_dev(), dtype=torch.bfloat16)
    p._tb_lp_shard = lp
    pr = torch.nn.Parameter(p0.clone())
    opt = FusedAdamW([p], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    ref = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    for _ in range(4):
        g = torch.randn(n, device=_dev()).to(gdtype)
        p._tb_grad = g
        pr.grad = g.float()
        opt.step()
        ref.step()
    _close(p, pr, 1e-4, 1e-5, "param")
    _close(lp, pr, 1e-2, 1e-2, "bf16 copy")


def test_sqnorm_and_clip_scale():
    from torchacc_b200.ops.optim import grad_sqnorm, scale_
    torch.manual_seed(0)
    gs = [torch.randn(12345, device=_dev()).bfloat16(), torch.randn(777, device=_dev())]
    stat = grad_sqnorm(gs)
    ref = sum((g.float() ** 2).sum() for g in gs)
    assert abs(float(stat[0]) - float(ref)) < 1e-3 * float(ref)
    assert float(stat[1]) == 0.0
    gs[1][5] = float("inf")
    assert float(grad_sqnorm(gs)[1]) == 1.0
    t = torch.ones(1000, device=_dev())
    scale_(t, torch.tensor([0.25], device=_dev()))
    assert torch.allclose(t, torch.full_like(t, 0.25))


def test_cpu_offload_moves_activations_and_preserves_grads():
    """reference tests/standalone/offload.py + utils/cpu_offload.py:521-605 on CUDA tensors: activations saved inside
    the offloaded groups really leave the device (pinned host buffers, D2H/H2D streams), memory drops, gradients are
    bit-identical to the non-offloaded run."""
    from torchacc_b200.utils.cpu_offload import get_cpu_offload_context
    torch.manual_seed(0)
    dev = _dev()
    layers = torch.nn.ModuleList([torch.nn.Sequential(torch.nn.Linear(2048, 2048), torch.nn.GELU(),
                                                      torch.nn.Linear(2048, 2048)) for _ in range(6)]).to(dev)
    x0 = torch.randn(4096, 2048, device=dev)

    def run(offload):
        for p in layers.parameters():
            p.grad = None
        x = x0.clone().requires_grad_()
        h = x
        if offload:
            ctx, sync = get_cpu_offload_context(num_offload_layers=4, num_prefetch_layers=1, num_offload_sync_layers=1)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for layer in layers:
            if offload:
                with ctx:
                    h = layer(h)
                h = sync(h)
            else:
                h = layer(h)
        if offload:
            ctx.offloader.finish_forward()
        torch.cuda.synchronize()
        mem_after_fwd = torch.cuda.memory_allocated()
        h.float().pow(2).mean().backward()
        torch.cuda.synchronize()
        grads = [p.grad.clone() for p in layers.parameters()] + [x.grad.clone()]
        return grads, mem_after_fwd, (ctx.offloader if offload else None)

    g_ref, mem_ref, _ = run(False)
    g_off, mem_off, off = run(True)
    assert off.offloaded_bytes >= 4 * 2 * 4096 * 2048 * 4, off.offloaded_bytes     # >= 2 saved activations x 4 groups
    assert off.d2h is not None and off.h2d is not None
    assert any(t.is_pinned() for lst in off.pool.free.values() for t in lst), "host buffers must be page-locked"
    assert mem_off < mem_ref - 3 * 4096 * 2048 * 4, (mem_off, mem_ref)              # device memory really dropped
    for a, b in zip(g_off, g_ref):
        assert torch.equal(a, b)


# ---- block-scaled fp8 ------------------------------------------------------------------------------------------------
def test_mxfp8_quantizer_matches_reference_and_layouts():
    from torchacc_b200.ops import fp8
    torch.manual_seed(0)
    x = (torch.randn(384, 512, device=_dev()) * torch.logspace(-3, 2, 512, device=_dev())).bfloat16()
    row, col = fp8.quantize_mxfp8(x, True, True)
    ref = fp8.quantize_mxfp8_ref(x)
    assert torch.equal(fp8.dequantize_mxfp8(row), ref), "row-wise payload / scale layout"
    ref_t = fp8.quantize_mxfp8_ref(x.t().contiguous())
    assert torch.equal(fp8.dequantize_mxfp8(col), ref_t), "transposed payload / scale layout"
    rel = (ref - x.float()).abs().max() / x.float().abs().max()
    assert rel < 0.07                                    # e4m3: 3 mantissa bits


@pytest.mark.parametrize("M,N,K", [(128, 192, 128), (256, 384, 512), (1000, 776, 384), (4096, 4096, 4096)])
def test_mxfp8_gemm_matches_fp32_oracle(M, N, K):
    """The kernel applies the UE8M0 block scales when it promotes each 32-element K block: D must equal the fp32 product
    of the DEQUANTISED operands, which pins the scale atom layout and the K-block selection (a wrong mapping is off by
    orders of magnitude).  Hopper's e4m3 MMA adds the 32 products of a K block in a datapath that keeps about 13
    fraction bits, so the result is not exact to fp32 rounding.  Observed on an H100, relative to the largest entry: 5.5e-5, 4.8e-5, 5.7e-5
    and 4.6e-5 for the four shapes; the bound is 1e-4."""
    from torchacc_b200.ops import fp8
    torch.manual_seed(1)
    # per-row and per-K-block magnitudes differ by orders of magnitude: a wrong scale mapping cannot hide
    a = (torch.randn(M, K, device=_dev()) * torch.logspace(-2, 2, M, device=_dev())[:, None]
         * (1 + torch.arange(K, device=_dev()) // 32 % 7)[None, :]).bfloat16()
    b = (torch.randn(N, K, device=_dev()) * torch.logspace(1, -2, N, device=_dev())[:, None]).bfloat16()
    aq, _ = fp8.quantize_mxfp8(a)
    bq, _ = fp8.quantize_mxfp8(b)
    d = fp8.gemm_mxfp8(aq, bq, out_dtype=torch.float32)
    ref = fp8.dequantize_mxfp8(aq).double() @ fp8.dequantize_mxfp8(bq).double().t()
    err = (d.double() - ref).abs().max() / ref.abs().max()
    assert err < 1e-4, float(err)
    # against the unquantised product: fp8 precision
    full = a.double() @ b.double().t()
    assert ((d.double() - full).norm() / full.norm()) < 0.06
    # bf16 output + addend
    c = torch.randn(M, N, device=_dev()).bfloat16()
    d2 = fp8.gemm_mxfp8(aq, bq, addend=c)
    _close(d2, ref.float() + c.float(), 2e-2, 2e-2 * float(ref.abs().max()), "bf16 out + addend")


def test_fp8_linear_fwd_bwd_close_to_bf16():
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops.linear import linear
    torch.manual_seed(2)
    T, K, N = 512, 1024, 768
    x = torch.randn(T, K, device=_dev()).bfloat16().requires_grad_()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16().requires_grad_()
    dy = torch.randn(T, N, device=_dev()).bfloat16()
    y0 = linear(x, w)
    y0.backward(dy)
    gx0, gw0 = x.grad.clone(), w.grad.clone()
    x.grad = w.grad = None
    fp8.enable(True)
    try:
        y1 = linear(x, w)
        y1.backward(dy)
    finally:
        fp8.enable(False)
    for a, b, what in ((y1, y0, "y"), (x.grad, gx0, "dx"), (w.grad, gw0, "dw")):
        rel = (a.float() - b.float()).norm() / b.float().norm()
        assert rel < 0.06, (what, float(rel))


# ---- fp16 operands on the native kernels (reference benchmark matrix is {bf16, fp16}: benchmarks/run.sh:8-48) -----------
def test_fp16_native_ops_match_fp32_reference():
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import rmsnorm
    from torchacc_b200.ops.swiglu import swiglu_separate
    from torchacc_b200.ops.linear import linear
    torch.manual_seed(0)
    dev = _dev()
    T, K, N = 512, 1024, 768
    x = (torch.randn(T, K, device=dev) * 0.5).half().requires_grad_()
    w = (torch.randn(N, K, device=dev) * 0.05).half().requires_grad_()
    b = torch.randn(N, device=dev).half().requires_grad_()
    n0 = nat.LAUNCHES
    y = linear(x, w, b)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert nat.LAUNCHES - n0 >= 3 and y.dtype == torch.float16
    xf, wf, bf = (t.detach().float().requires_grad_() for t in (x, w, b))
    yr = F.linear(xf, wf, bf)
    yr.backward(dy.float())
    _close(y, yr, 4e-3, 4e-3 * float(yr.abs().max()), "fp16 linear fwd")
    _close(x.grad, xf.grad, 4e-3, 4e-3 * float(xf.grad.abs().max()), "fp16 dgrad")
    _close(w.grad, wf.grad, 4e-3, 4e-3 * float(wf.grad.abs().max()), "fp16 wgrad")
    # rmsnorm + residual, swiglu
    h = torch.randn(T, K, device=dev).half().requires_grad_()
    res = torch.randn(T, K, device=dev).half()
    g = (torch.rand(K, device=dev) + 0.5).half().requires_grad_()
    n0 = nat.LAUNCHES
    yn, hn = rmsnorm(h, g, 1e-5, residual=res)
    yn.float().square().sum().backward()
    assert nat.LAUNCHES - n0 >= 2 and yn.dtype == torch.float16
    hf, gf = h.detach().float().requires_grad_(), g.detach().float().requires_grad_()
    s = hf + res.float()
    yr = s * torch.rsqrt(s.pow(2).mean(-1, keepdim=True) + 1e-5) * gf
    yr.square().sum().backward()
    _close(yn, yr, 1e-2, 1e-2, "fp16 rmsnorm")        # the kernel normalises the fp16-rounded residual stream
    _close(h.grad, hf.grad, 3e-2, 3e-2 * float(hf.grad.abs().max()), "fp16 rmsnorm dx")
    gate, up = torch.randn(T, N, device=dev).half().requires_grad_(), torch.randn(T, N, device=dev).half().requires_grad_()
    n0 = nat.LAUNCHES
    o = swiglu_separate(gate, up)
    o.float().sum().backward()
    assert nat.LAUNCHES - n0 >= 2 and o.dtype == torch.float16
    gr, ur = gate.detach().float().requires_grad_(), up.detach().float().requires_grad_()
    (F.silu(gr) * ur).sum().backward()
    _close(o, F.silu(gr) * ur, 4e-3, 4e-3, "fp16 swiglu")
    _close(gate.grad, gr.grad, 6e-3, 6e-3, "fp16 swiglu dgate")


def test_gate_up_swiglu_epilogue_matches_separate_ops():
    """gate|up GEMM with the SwiGLU activation in its epilogue vs GEMM + swiglu kernel: forward, and backward through
    the kept pre-activation; also the checkpointed form (first pass skips the [T, 2F] write, recompute provides it)."""
    from torch.utils.checkpoint import checkpoint
    from torchacc_b200.ops.linear import linear
    from torchacc_b200.ops.swiglu import activations_recomputed_later, gate_up_swiglu, swiglu
    torch.manual_seed(3)
    T, K, Fd = 640, 512, 1280                       # T not a multiple of 256: ragged last M tile
    x = (torch.randn(T, K, device=_dev()) * 0.7).bfloat16().requires_grad_()
    w = (torch.randn(2 * Fd, K, device=_dev()) * 0.06).bfloat16().requires_grad_()
    dh = torch.randn(T, Fd, device=_dev()).bfloat16()
    h0 = swiglu(linear(x, w))
    h0.backward(dh)
    gx0, gw0 = x.grad.clone(), w.grad.clone()
    x.grad = w.grad = None
    h1 = gate_up_swiglu(x, w)
    _close(h1, h0, 2e-2, 2e-2, "fused fwd")          # fused applies silu to the fp32 accumulators (slightly more exact)
    h1.backward(dh)
    _close(x.grad, gx0, 2e-2, 2e-2 * float(gx0.abs().max()), "fused dx")
    _close(w.grad, gw0, 2e-2, 2e-2 * float(gw0.abs().max()), "fused dw")
    # fp32 oracle for the forward
    g, u = (x.float() @ w.float().t()).chunk(2, -1)
    _close(h1, F.silu(g) * u, 2e-2, 2e-2, "fused fwd vs fp32")
    # checkpointed: the first pass runs with the flag set (no pre-activation written), backward recomputes
    x.grad = w.grad = None

    def f(a, b):
        return gate_up_swiglu(a, b)
    with activations_recomputed_later():
        h2 = checkpoint(f, x, w, use_reentrant=False)
    h2.backward(dh)
    assert torch.equal(h2, h1)
    _close(x.grad, gx0, 2e-2, 2e-2 * float(gx0.abs().max()), "ckpt dx")
    _close(w.grad, gw0, 2e-2, 2e-2 * float(gw0.abs().max()), "ckpt dw")
