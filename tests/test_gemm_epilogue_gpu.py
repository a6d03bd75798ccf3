"""The dense GEMM's staged epilogue (csrc/gemm/gemm_bf16.cu, kStaged): registers -> swizzled shared memory -> TMA store
(TMA-loaded 16-bit addend, TMA reduce-add for fp32 accumulation).  The host picks it for 16-byte aligned outputs and
keeps the register epilogue for anything else, so the same GEMM into an aligned D and into a D one element off must
give bitwise the same results, under static and dynamic tile scheduling, and both must match an fp32 reference."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _sched(mode):
    from torchacc_b200 import _native as nat
    L = nat.require()
    prev = L.tb_gemm_sched_mode(-1)
    L.tb_gemm_sched_mode(1 if mode == "dynamic" else 0)
    return lambda: L.tb_gemm_sched_mode(prev)


def _bitwise(a, b, what=""):
    assert a.dtype == b.dtype and a.shape == b.shape
    bits = {2: torch.int16, 4: torch.int32}[a.element_size()]
    bad = (a.view(bits) != b.view(bits)).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} elements differ between the staged and the register epilogue"


def _close(a, ref, K, what=""):
    a = a.float()
    tol = 2e-2 * ref.abs() + 2e-3 * math.sqrt(K) + 1e-2
    bad = ((a - ref).abs() > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches against fp32, max err {(a - ref).abs().max().item():.4g}"


def _pitch(cols):   # a padded row pitch: a multiple of 16 bytes for 16-bit and fp32 elements, wider than the matrix
    return (cols + 7) // 8 * 8 + 8


def _operands(M, N, K, a_mn, b_mn, dtype, seed=0):
    g = torch.Generator(device=_dev()).manual_seed(seed)

    def operand(rows, cols):
        return torch.randn(rows, _pitch(cols), device=_dev(), generator=g).to(dtype)[:, :cols]
    a = operand(K, M) if a_mn else operand(M, K)
    b = operand(K, N) if b_mn else operand(N, K)
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    return a, b, A @ B


def _out_pair(M, N, dtype, init=None):
    """Two [M, N] views with the same padded pitch: one 16-byte aligned (staged epilogue), one a single element off
    (register epilogue).  Both start from `init` when given."""
    pitch = _pitch(N)
    outs = []
    for off in (0, 1):
        buf = torch.zeros(M * pitch + 8, dtype=dtype, device=_dev())
        o = buf[off:off + M * pitch].view(M, pitch)[:, :N]
        if init is not None:
            o.copy_(init)
        outs.append(o)
    return outs


@pytest.mark.parametrize("sched", ["static", "dynamic"])
@pytest.mark.parametrize("shape", [(328, 328, 136), (77, 520, 200)])   # ragged M and N tiles
@pytest.mark.parametrize("mode", ["bf16", "fp16", "bias", "addend", "acc16", "fp32_out", "fp32_bias", "fp32_acc_view"])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (1, 1)])
def test_staged_matches_register(a_mn, b_mn, mode, shape, sched):
    from torchacc_b200.ops.linear import gemm
    M, N, K = shape
    dtype = torch.float16 if mode == "fp16" else torch.bfloat16
    a, b, ref = _operands(M, N, K, a_mn, b_mn, dtype, seed=1)
    g = torch.Generator(device=_dev()).manual_seed(2)
    bias = torch.randn(N, device=_dev(), generator=g).to(dtype)
    addend = torch.randn(M, _pitch(N), device=_dev(), generator=g).to(dtype)[:, :N]
    init16 = torch.randn(M, N, device=_dev(), generator=g).to(dtype)
    kw = dict(a_mn_major=bool(a_mn), b_mn_major=bool(b_mn))
    restore = _sched(sched)
    try:
        if mode == "fp32_acc_view":
            # an fp32 gradient buffer, D a strided view at an offset of 8 elements (staged) or 9 (register)
            init = torch.randn(M, N, device=_dev(), generator=g)
            outs = []
            for off in (8, 9):
                view = torch.zeros(M, N + 24, device=_dev())[:, off:off + N]
                view.copy_(init)
                gemm(a, b, out=view, accumulate=True, **kw)
                outs.append(view)
            expect = init + ref
        elif mode.startswith("fp32"):
            outs = _out_pair(M, N, torch.float32)
            for o in outs:
                gemm(a, b, out=o, bias=bias if mode == "fp32_bias" else None, **kw)
            expect = ref + (bias.float() if mode == "fp32_bias" else 0)
        elif mode == "acc16":
            outs = _out_pair(M, N, dtype, init=init16)
            for o in outs:
                gemm(a, b, out=o, accumulate=True, **kw)
            expect = ref + init16.float()
        else:
            outs = _out_pair(M, N, dtype)
            for o in outs:
                gemm(a, b, out=o, bias=bias if mode == "bias" else None,
                     addend=addend if mode == "addend" else None, **kw)
            expect = ref + (bias.float() if mode == "bias" else 0) + (addend.float() if mode == "addend" else 0)
        torch.cuda.synchronize()
    finally:
        restore()
    assert outs[0].data_ptr() % 16 == 0 and outs[1].data_ptr() % 16 != 0
    _bitwise(outs[0], outs[1], f"{mode} {shape} {sched}")
    _close(outs[0], expect, K, f"{mode} vs fp32")


@pytest.mark.parametrize("write_gu", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_staged_swiglu(write_gu, dtype):
    """The SwiGLU epilogue always stages.  g|u must be bitwise the plain GEMM's register-epilogue output (same
    accumulation order per element), h must match silu(g) * u of the fp32 reference."""
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops.linear import gemm
    L = nat.require()
    M, F, K = 200, 384, 264
    g = torch.Generator(device=_dev()).manual_seed(3)
    x = torch.randn(M, K, device=_dev(), generator=g).to(dtype)
    w = (torch.randn(2 * F, K, device=_dev(), generator=g) / 4).to(dtype)
    h = torch.full((M, F), 7.0, device=_dev(), dtype=dtype)
    gu = torch.full((M, 2 * F), 7.0, device=_dev(), dtype=dtype)
    nat.check(L.tb_gemm_swiglu(x.data_ptr(), w.data_ptr(), h.data_ptr(), gu.data_ptr() if write_gu else 0, M, F, K,
                               K, K, F, 2 * F, nat.num_sms(), nat.stream(), int(dtype == torch.float16)),
              "tb_gemm_swiglu")
    _, plain = _out_pair(M, 2 * F, dtype)   # misaligned: the register epilogue
    gemm(x, w, out=plain)
    torch.cuda.synchronize()
    if write_gu:
        _bitwise(gu, plain, "g|u")
    else:
        assert (gu == 7.0).all(), "g|u was written although it was not requested"
    ref = x.float() @ w.float().t()
    hg, hu = ref[:, :F], ref[:, F:]
    _close(h, torch.nn.functional.silu(hg) * hu, K, "h vs fp32")


def test_staged_lm_head_dw():
    """The LM-head weight gradient of the flagship (128256 x 2048 x 4096, fp32, accumulated over two chunks): the
    TMA reduce-add against the register epilogue."""
    from torchacc_b200.ops.linear import gemm
    V, H, T = 128256, 2048, 4096
    g = torch.Generator(device=_dev()).manual_seed(6)
    lg = (torch.randn(T, V, device=_dev(), generator=g) / 16).bfloat16()
    hid = torch.randn(T, H, device=_dev(), generator=g).bfloat16()
    outs = []
    for off in (0, 1):
        buf = torch.zeros(V * H + 4, device=_dev())
        dw = buf[off:off + V * H].view(V, H)
        for _ in range(2):
            gemm(lg, hid, a_mn_major=True, b_mn_major=True, out=dw, accumulate=True)
        outs.append(dw)
    torch.cuda.synchronize()
    assert outs[0].data_ptr() % 16 == 0 and outs[1].data_ptr() % 16 != 0
    _bitwise(outs[0], outs[1], "LM-head dW")
    rows = torch.arange(0, V, 997, device=_dev())
    ref = 2 * (lg[:, rows].float().t() @ hid.float())
    _close(outs[0][rows], ref, T, "LM-head dW vs fp32")
