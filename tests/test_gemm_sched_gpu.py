"""The dense GEMM without a carried collective (csrc/gemm/gemm_bf16.cu, kCarry == false) under static and dynamic tile
scheduling: a tile's accumulation order does not depend on which CTA computes it, so both grids must give bitwise the
same results, and those results must match an fp32 reference."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _lib():
    from torchacc_b200 import _native as nat
    return nat.require()


def _both_modes(fn):
    """fn() once under static (persistent grid) and once under dynamic (one CTA per tile) scheduling."""
    L = _lib()
    prev = L.tb_gemm_sched_mode(-1)
    try:
        L.tb_gemm_sched_mode(0)
        static = fn()
        L.tb_gemm_sched_mode(1)
        dynamic = fn()
        torch.cuda.synchronize()
    finally:
        L.tb_gemm_sched_mode(prev)
    return static, dynamic


def _bitwise(a, b, what=""):
    assert a.dtype == b.dtype and a.shape == b.shape
    bits = {2: torch.int16, 4: torch.int32}[a.element_size()]
    bad = (a.view(bits) != b.view(bits)).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} elements differ between static and dynamic scheduling"


def _close(a, ref, K, what=""):
    a = a.float()
    tol = 2e-2 * ref.abs() + 2e-3 * math.sqrt(K) + 1e-2
    bad = ((a - ref).abs() > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches against fp32, max err {(a - ref).abs().max().item():.4g}"


def _operands(M, N, K, a_mn, b_mn, dtype, seed=0):
    g = torch.Generator(device=_dev()).manual_seed(seed)

    def operand(rows, cols):   # row pitch padded to 16 bytes (TMA), e.g. an MN-major A with M = 77
        pitch = (cols + 7) // 8 * 8
        return torch.randn(rows, pitch, device=_dev(), generator=g).to(dtype)[:, :cols]
    a = operand(K, M) if a_mn else operand(M, K)
    b = operand(K, N) if b_mn else operand(N, K)
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    return a, b, A @ B   # reference [M, N]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("M", [77, 328, 1000])   # 1, 3 and 8 M tiles
def test_sched_bitwise_majors(M, a_mn, b_mn, dtype):
    from torchacc_b200.ops.linear import gemm
    N, K = 328, 136
    a, b, ref = _operands(M, N, K, a_mn, b_mn, dtype)
    static, dynamic = _both_modes(lambda: gemm(a, b, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn)))
    _bitwise(static, dynamic, f"M={M} a_mn={a_mn} b_mn={b_mn} {dtype}")
    if M == 328:
        _close(dynamic, ref, K, "vs fp32")


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (1, 1)])
@pytest.mark.parametrize("mode", ["fp32_out", "fp32_acc_view", "bias", "addend", "acc16"])
def test_sched_bitwise_epilogues(mode, a_mn, b_mn):
    from torchacc_b200.ops.linear import gemm
    M, N, K = 328, 328, 136
    a, b, ref = _operands(M, N, K, a_mn, b_mn, torch.bfloat16, seed=1)
    g = torch.Generator(device=_dev()).manual_seed(2)
    bias = torch.randn(N, device=_dev(), generator=g).bfloat16()
    addend = torch.randn(M, N, device=_dev(), generator=g).bfloat16()
    base32 = torch.randn(M, N + 24, device=_dev(), generator=g)   # fp32 gradient buffer, D a strided view of it
    base16 = torch.randn(M, N, device=_dev(), generator=g).bfloat16()

    def run():
        kw = dict(a_mn_major=bool(a_mn), b_mn_major=bool(b_mn))
        if mode == "fp32_out":
            return gemm(a, b, out_dtype=torch.float32, **kw)
        if mode == "fp32_acc_view":
            buf = base32.clone()
            gemm(a, b, out=buf[:, 8:8 + N], accumulate=True, **kw)
            return buf
        if mode == "bias":
            return gemm(a, b, bias=bias, **kw)
        if mode == "addend":
            return gemm(a, b, addend=addend, **kw)
        out = base16.clone()
        gemm(a, b, out=out, accumulate=True, **kw)
        return out

    static, dynamic = _both_modes(run)
    _bitwise(static, dynamic, mode)
    expect = {"fp32_out": ref, "bias": ref + bias.float(), "addend": ref + addend.float(),
              "acc16": ref + base16.float()}.get(mode)
    if mode == "fp32_acc_view":
        expect = base32.clone()
        expect[:, 8:8 + N] += ref
    _close(dynamic, expect, K, f"{mode} vs fp32")


@pytest.mark.parametrize("case", ["persistent", "wgrad_qkv"])
def test_sched_bitwise_large(case):
    """Many tiles per CTA of the persistent grid, and the flagship wgrad of the QKV projection (fp32, accumulated)."""
    from torchacc_b200.ops.linear import gemm
    if case == "persistent":
        a, b, _ = _operands(8192, 4096, 2048, 0, 0, torch.bfloat16, seed=4)
        static, dynamic = _both_modes(lambda: gemm(a, b))
    else:
        a, b, _ = _operands(3072, 2048, 8192, 1, 1, torch.bfloat16, seed=5)
        init = torch.randn(3072, 2048, device=_dev())

        def run():
            out = init.clone()
            gemm(a, b, a_mn_major=True, b_mn_major=True, out=out, accumulate=True)
            return out
        static, dynamic = _both_modes(run)
    _bitwise(static, dynamic, case)
