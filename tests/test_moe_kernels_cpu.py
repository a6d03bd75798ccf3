"""CPU tier of ``test_moe_kernels_gpu.py``: its oracles agree with independent references, and its checkers reject
planted faults in PyTorch emulations of the kernels."""
import pytest
import torch

from test_moe_kernels_gpu import (BF16, FP16, FP32, ROUND, U8, check_index, check_permute, combine_ref,
                                  e4m3_round, emulate_combine_fwd, emulate_permute, emulate_unpermute_sum,
                                  expect_equal, expect_rounded, index_oracle, mx_oracle, pow2, router_oracle, router_premise,
                                  scale_bytes)


def test_e4m3_oracle_matches_torch_cast():
    """Every bf16 value with |x| <= 448, and a dense fp32 sample of [-448, 448] incl. every midpoint between e4m3
    neighbours (the ties) and the subnormal range, round as torch.float8_e4m3fn does."""
    allb = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16)
    x = allb[allb.float().abs() <= 448].float()
    table = torch.tensor(sorted(set(torch.arange(0, 127, dtype=U8).view(torch.float8_e4m3fn).float().tolist())),
                         dtype=FP32)
    mids = (table[1:] + table[:-1]) / 2
    dense = torch.linspace(-448, 448, 2_000_001)
    tiny = torch.linspace(-2.0 ** -5, 2.0 ** -5, 200_001)
    for v in (x, torch.cat([mids, -mids, dense, tiny])):
        expect_equal(e4m3_round(v.double()), v.to(torch.float8_e4m3fn).view(U8), "e4m3 oracle vs torch")


def _kernel_scale_formula(amax, round_up=True):
    """csrc/ops/quant_mxfp8.cu ``e8m0_from_amax`` emulated in fp32 (``round_up=False``: a planted fault)."""
    x = (amax.float() * torch.tensor(1.0 / 448.0, dtype=FP32)).view(torch.int32)
    e = (x >> 23) & 0xFF
    if round_up:
        e = e + ((x & 0x7FFFFF) != 0).int()
    e = torch.where(e == 0, torch.ones_like(e), e).clamp(max=254)
    return torch.where(amax.float() > 0, e, torch.zeros_like(e)).long()


@pytest.mark.parametrize("fault", ["none", "exponent_not_rounded_up"])
def test_scale_byte_oracle(fault):
    """The integer scale-byte oracle equals the kernel's fp32 formula on every positive bf16 amax; the formula without
    the exponent round-up is rejected."""
    amax = torch.arange(0, 0x7F81, dtype=torch.int32).to(torch.int16).view(BF16)
    got = _kernel_scale_formula(amax, round_up=fault == "none")
    if fault == "none":
        expect_equal(got, scale_bytes(amax), "scale byte")
        assert int(scale_bytes(amax[-2:-1])) == 247
    else:
        with pytest.raises(AssertionError):
            expect_equal(got, scale_bytes(amax), "scale byte")


def test_quantize_mxfp8_ref_follows_the_kernel_on_non_finite_blocks():
    """``quantize_mxfp8_ref`` (the op's PyTorch emulation) gives the oracle's values, NaN / inf blocks included."""
    from torchacc_b200.ops import fp8
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(16, 256, generator=g) * torch.exp2(torch.randint(-30, 30, (16, 1), generator=g).float())).to(BF16)
    x[1, 5] = float("nan")
    x[2, 70] = float("inf")
    x[3, 33] = -float("inf")
    x[4, 64:96] = float("nan")
    x[5, 0:32] = 0
    codes, scales = mx_oracle(x)
    vals = codes.view(torch.float8_e4m3fn).double() * pow2(scales - 127).repeat_interleave(32, 1)
    expect_equal(fp8.quantize_mxfp8_ref(x).double(), vals, "quantize_mxfp8_ref vs the oracle")
    assert bool(torch.isnan(vals[1, 5])) and int(torch.isnan(vals[1]).sum()) == 1
    assert bool(torch.isnan(vals[2, 70])) and bool((vals[2, 64:96].nan_to_num(1.0) == 0).sum() == 31)


def test_router_oracle_matches_reference():
    from torchacc_b200.ops.moe import moe_router_reference
    g = torch.Generator().manual_seed(1)
    for E, k in ((8, 2), (60, 4), (256, 8)):
        z = torch.rand(300, E, generator=g).argsort(-1).float() / 16 - E / 32   # distinct in each row: no ties
        p, ids = router_oracle(z, k)
        router_premise(p, k, "reference data")
        for norm in (False, True):
            w, idr = moe_router_reference(z, k, norm)
            expect_equal(ids, idr, "router oracle ids")
            pj = p.gather(-1, ids)
            w64 = pj / pj.sum(-1, keepdim=True) if norm else pj
            assert torch.allclose(w.double(), w64, rtol=1e-6, atol=0)


@pytest.mark.parametrize("fault", ["none", "tie_to_higher_index"])
def test_router_checker_rejects_ties_to_the_higher_index(fault):
    g = torch.Generator().manual_seed(2)
    z = torch.randint(-3, 4, (64, 60), generator=g).to(BF16) * 0.5
    p, want = router_oracle(z, 8)
    key = p.double()
    if fault == "none":
        got = torch.sort(key, dim=-1, descending=True, stable=True).indices[:, :8]
        expect_equal(got, want, "ids")
    else:   # sort the reversed row: equal values come out highest index first
        got = (59 - torch.sort(key.flip(-1), dim=-1, descending=True, stable=True).indices)[:, :8]
        with pytest.raises(AssertionError):
            expect_equal(got, want, "ids")


def _layout(T=700, k=4, E=16, seed=3):
    from torchacc_b200.ops.moe import capacity
    g = torch.Generator().manual_seed(seed)
    ids = torch.rand(T, E, generator=g).argsort(-1)[:, :k]
    ids[::5, k - 1] = E
    ids[::7, 0] = -1
    rows = capacity(T, k, E)
    return ids, E, rows, index_oracle(ids, E, rows), g


@pytest.mark.parametrize("fault", ["none", "rank_off_by_one_across_a_round"])
def test_index_checker(fault):
    ids, E, rows, (counts, offsets, te, tiles, pos, row_src), _ = _layout()
    pos, row_src = pos.clone(), row_src.clone()
    got = [counts, offsets, te, tiles, pos, row_src]
    if fault == "none":
        check_index(got, ids, E, rows, "oracle against itself")
        return
    i = ROUND + int((pos[ROUND:] >= 0).nonzero()[0])   # first routed entry of the second round
    pos[i] += 1                                        # its rank counted one too many earlier entries
    with pytest.raises(AssertionError):
        check_index(got, ids, E, rows, "planted fault")


@pytest.mark.parametrize("fault", ["none", "padding_row_not_zeroed"])
def test_permute_checker(fault):
    """The permute emulation agrees with ``_sorted_layout``: unpermuting the permuted rows gives every token times its
    number of routed slots; a padding row left unzeroed is rejected."""
    ids, E, rows, (counts, offsets, te, tiles, pos, row_src), g = _layout()
    k = ids.shape[1]
    x = torch.randn(ids.shape[0], 64, generator=g).to(BF16)
    xp = torch.full((rows, 64), float("nan"), dtype=BF16)
    emulate_permute(x, row_src, offsets, k, xp)
    if fault == "none":
        check_permute(xp, x, row_src, offsets, k, "emulation")
        n = (pos.view(ids.shape) >= 0).sum(1, keepdim=True)
        expect_equal(emulate_unpermute_sum(xp, pos.view(ids.shape)), (x.float() * n).to(BF16), "unpermute(permute)")
        assert bool(torch.isnan(xp[int(offsets[-1]):]).all())
    else:
        pad = int((row_src[:int(offsets[-1])] < 0).nonzero()[0])
        xp[pad] = x[0]
        with pytest.raises(AssertionError):
            check_permute(xp, x, row_src, offsets, k, "planted fault")


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("fault", ["none", "residual_before_rounding", "residual_in_loop", "weights_16bit"])
def test_combine_checker(fault, dtype):
    """The exact combine case of the GPU tests (integer rows, weights on a 2^-12 grid, integer residual): the emulated
    kernel is the single rounding of the fp64 result, and every planted fault is rejected."""
    ids, E, rows, (counts, offsets, te, tiles, pos, row_src), g = _layout(k=8)
    T, k = ids.shape
    pos = pos.view(T, k)
    y = torch.randint(-64, 65, (rows, 64), generator=g).to(dtype)
    w = torch.randint(-4096, 4097, (T, k), generator=g).float() / 4096
    res = torch.randint(-1000, 1001, (T, 64), generator=g).to(dtype)
    ref, _ = combine_ref(y, pos, w, res)
    out = emulate_combine_fwd(y, pos, w, res, None if fault == "none" else fault)
    if fault == "none":
        expect_rounded(out, ref, "emulated combine")
    else:
        with pytest.raises(AssertionError):
            expect_rounded(out, ref, f"planted fault {fault}")
