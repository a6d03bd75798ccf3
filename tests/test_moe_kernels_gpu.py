"""The MoE routing kernels (csrc/ops/moe.cu: router forward / backward, index build, permute, unpermute-sum, combine
forward / backward) and the MX-FP8 quantiser (csrc/ops/quant_mxfp8.cu) against fp64 references.

Exact checks (``==``, NaN fails) wherever the arithmetic allows it; each test asserts its exactness premise:
  - router ids: experts ranked by fp64 probability, ties to the lower index.  Premise (``router_premise``): among the
    k + 1 best experts of a row, distinct probabilities differ by far more than the kernel's fp32 error, and every fp64
    probability is either a normal fp32 number or so small that fp32 expf gives exactly 0 (those tie at 0);
  - index build: ``ops/moe.py::_sorted_layout`` plus counts, offsets, tile owners, tile count and row sources;
  - permute and combine backward's d(y_perm): bitwise copies / the kernel's two-step rounding;
  - unpermute-sum and combine forward on small integers and dyadic weights, where every fp32 step is exact: the output
    is the single 16-bit rounding of the fp64 result;
  - the quantiser: payload and scale bytes against an oracle that never uses torch's float8 cast (scale byte by integer
    arithmetic on the bf16 bits, elements rounded to nearest-even against the 256-entry e4m3 table).
Everything else is compared with fp64 under a bound derived from the kernel's arithmetic, written next to each check and
printed as ``[bound]`` lines with the fraction used.  u = 2^-24 is the fp32 unit roundoff.  The bounds are first-order
sums of per-operation errors; each is multiplied by (1 + 2^-10), which covers the second-order terms (all O(u) relative
to the first-order ones).

Every output sits inside a buffer of sentinel bits (``Guarded``) that must survive where the kernel must not write.

``test_moe_kernels_cpu.py`` runs the oracles and checkers of this file without a GPU, and shows that they reject
planted faults in emulated kernels."""
import math

import pytest
import torch

from test_gemm_kernels_gpu import ulp_dtype

gpu = pytest.mark.gpu
DEV = "cuda"
BF16, FP16, FP32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
I32, I64, U8 = torch.int32, torch.int64, torch.uint8
U = 2.0 ** -24                      # fp32 unit roundoff
SECOND_ORDER = 1 + 2.0 ** -10
TILE = 128
ROUND = 1024                        # entries per round of the index build


# ---------------------------------------------------------------------------------------------------------------------
# guarded outputs and checkers (device agnostic)
# ---------------------------------------------------------------------------------------------------------------------
_INT_OF = {1: U8, 2: torch.int16, 4: I32, 8: I64}
_SENTINEL = {FP32: 0x7FC05A5A, BF16: 0x7FA5, FP16: 0x7E5A, I64: -0x5A5A5A5A5A5A5A5B, I32: -0x5A5A5A5B, U8: 0xA5}


def _esz(dtype):
    return torch.empty((), dtype=dtype).element_size()


def bits(t):
    return t.view(_INT_OF[_esz(t.dtype)])


class Guarded:
    """A contiguous ``shape`` output ``view`` on a 16-byte aligned base, with ``pad`` sentinel elements before and after
    (NaN bits no kernel produces for float outputs); the view starts out holding sentinels too."""

    def __init__(self, shape, dtype, pad=64, device=DEV):
        n = math.prod(shape)
        self.dtype, self.pad, self.n = dtype, pad, n
        self.buf = torch.full((n + 2 * pad,), _SENTINEL[dtype], dtype=_INT_OF[_esz(dtype)], device=device).view(dtype)
        self.view = self.buf[pad:pad + n].view(shape)

    def sentinel(self):
        """True where the view still holds the sentinel bits."""
        return bits(self.view) == _SENTINEL[self.dtype]

    def check_untouched(self, what, mask=None):
        """The pads, and the view elements where ``mask`` is True, still hold the sentinel bits."""
        b = bits(self.buf)
        s = _SENTINEL[self.dtype]
        n = int((b[:self.pad] != s).sum()) + int((b[self.pad + self.n:] != s).sum())
        assert n == 0, f"{what}: {n} sentinel elements around the output were written"
        if mask is not None:
            n = int((mask & ~self.sentinel()).sum())
            assert n == 0, f"{what}: {n} elements the kernel must not write were written"


def padded_input(vals, poison=float("nan"), pad=64):
    """``vals`` copied into a 16-byte aligned, contiguous view with ``pad`` poison elements on each side: a read past it
    poisons the result."""
    flat = torch.full((vals.numel() + 2 * pad,), poison, dtype=vals.dtype, device=vals.device)
    v = flat[pad:pad + vals.numel()].view(vals.shape)
    v.copy_(vals)
    return v


def expect_equal(out, want, what):
    """Bitwise equality (for floats, NaN matches NaN only where both are NaN)."""
    assert out.shape == want.shape, (what, tuple(out.shape), tuple(want.shape))
    if out.dtype.is_floating_point:
        bad = ~((out == want) | (torch.isnan(out) & torch.isnan(want)))
        bad |= (out == 0) & (want == 0) & (torch.signbit(out) != torch.signbit(want))
    else:
        bad = out != want
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} elements differ; first at {idx}: out "
                             f"{out[tuple(idx)].item()!r} want {want[tuple(idx)].item()!r}")


def expect_rounded(out, ref64, what):
    """``out`` equals the single rounding of the exact fp64 result to its dtype (NaN fails)."""
    want = ref64.to(out.dtype)
    bad = torch.isnan(out) | (out.double() != want.double())
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} elements differ from the single rounding of the "
                             f"fp64 result; first at {idx}: out {out[tuple(idx)].item()!r} want "
                             f"{want[tuple(idx)].item()!r} (exact {ref64[tuple(idx)].item()!r})")


def within(out, ref64, bound, what):
    """|out - ref| <= bound everywhere (NaN fails); prints the largest fraction of the bound used."""
    err = (out.double() - ref64).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} outside the derived bound; first at flat index "
                             f"{i}: out {out.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r} bound "
                             f"{bound.reshape(-1)[i].item() if torch.is_tensor(bound) else bound!r}")
    used = float((err / bound).nan_to_num(0.0).max()) if out.numel() else 0.0
    print(f"[bound] {what}: {used:.3f} of the bound")
    return used


def half_ulp(ref64, err, dtype):
    """Half an ulp of ``dtype`` where a value within ``err`` of ``ref64`` rounds (fp32: covered by the fp32 terms)."""
    if dtype == FP32:
        return torch.zeros_like(ref64)
    return 0.5 * ulp_dtype(ref64.abs() + err, dtype)


# ---------------------------------------------------------------------------------------------------------------------
# router oracle
# ---------------------------------------------------------------------------------------------------------------------
TINY_ZERO = 2.0 ** -155     # fp64 probabilities below this are exactly 0 in the kernel (expf < 2^-150 rounds to 0)
TINY_NORMAL = 2.0 ** -100   # above this the kernel's fp32 probability is a normal number with a small relative error
UNDERFLOW = 2.0 ** -148     # absolute error of a probability that underflows: expf and the product each round to 2^-150


def bad_rows(z):
    """Rows whose softmax the kernel turns into NaN: a NaN or +inf logit, or every logit -inf."""
    return torch.isnan(z).any(-1) | (z == float("inf")).any(-1) | (z == float("-inf")).all(-1)


def router_oracle(logits, k):
    """(p64 [T, E] (NaN on bad rows), ids [T, k] int64): experts ranked by fp64 probability, ties to the lower index;
    NaN ranks above every number (torch.topk's order), so a bad row picks experts 0..k-1."""
    z = logits.double()
    bad = bad_rows(z)
    p = torch.softmax(torch.where(bad[:, None], torch.zeros_like(z), z), -1)
    p = torch.where(bad[:, None], torch.full_like(p, float("nan")), p)
    key = torch.where(p < TINY_ZERO, torch.zeros_like(p), p)
    key = torch.where(bad[:, None], torch.ones_like(key), key)
    ids = torch.sort(key, dim=-1, descending=True, stable=True).indices[:, :k]
    return p, ids


def router_rel_err(z, p):
    """Relative error bound of the kernel's fp32 probabilities, per element: z - max rounds (|z - m| u, which moves
    exp by that relative amount), expf <= 2 ulp (4u), the sum of E terms (each lane's serial sum of <= 8, then 5
    butterfly levels: <= 13 roundings, on top of the worst term error), the reciprocal (u) and the product (u)."""
    zf = torch.where(torch.isfinite(z), z, torch.full_like(z, float("-inf")))
    m = zf.max(-1, keepdim=True).values
    d = torch.where(torch.isfinite(zf), (zf - m).abs(), torch.zeros_like(zf))
    term = (4 + d) * U
    return term + term.max(-1, keepdim=True).values + 15 * U


def router_premise(p, k, what):
    """Among the k + 1 best experts of each good row: every fp64 probability is 0 for the kernel (< TINY_ZERO) or a
    normal fp32 number (> TINY_NORMAL), and distinct ones differ by a ratio of more than 1 + 2^-12, far above twice the
    kernel's relative error (router_rel_err, < 2^-15 here)."""
    good = ~torch.isnan(p).any(-1)
    s = torch.sort(p[good], -1, descending=True).values[:, :min(k + 1, p.shape[1])]
    assert not bool(((s >= TINY_ZERO) & (s <= TINY_NORMAL)).any()), f"{what}: a probability in the ambiguous range"
    a, b = s[:, :-1], s[:, 1:]
    close = (a != b) & (b > TINY_NORMAL) & (a <= b * (1 + 2.0 ** -12))
    assert not bool(close.any()), f"{what}: two top-{k} probabilities too close to order by an fp32 computation"


def router_weights_bound(z, p, ids, norm):
    """(w64, bound) for the chosen experts: w_j = p_j, or p_j / S with S the k-term sum in selection order ((k - 1)
    roundings) and one IEEE division."""
    rel = router_rel_err(z, p).gather(-1, ids)
    pj = p.gather(-1, ids)
    if not norm:
        return pj, (rel * pj * SECOND_ORDER + UNDERFLOW)
    S = pj.sum(-1, keepdim=True)
    w = pj / S
    relS = rel.max(-1, keepdim=True).values + (ids.shape[1] - 1) * U
    return w, (rel + relS + U) * w * SECOND_ORDER + UNDERFLOW


def router_dlogits_bound(z, p, ids, dw, norm, out_dtype):
    """(dz64, bound) for the backward's formula at the chosen ids (see the kernel's comment):
        S = sum_j p_j;  dot = sum_j dw_j p_j / S;  g_j = (dw_j - dot) / S (norm) or dw_j;  pg = sum_j p_j g_j;
        dz_m = p_m (g_m - pg)
    with absolute error bounds carried through every fp32 operation in the kernel's order (first order), plus half an
    ulp of a 16-bit output."""
    dw = dw.double()
    ep = router_rel_err(z, p) * p + UNDERFLOW           # |p_hat - p|
    pj, epj = p.gather(-1, ids), ep.gather(-1, ids)
    k = ids.shape[1]
    S = pj.sum(-1, keepdim=True)
    eS = epj.sum(-1, keepdim=True) + (k - 1) * U * S
    t = dw * pj / S
    et = dw.abs() * (epj / S + pj * eS / S ** 2) + 2 * U * t.abs()
    dot = t.sum(-1, keepdim=True)
    edot = et.sum(-1, keepdim=True) + (k - 1) * U * t.abs().sum(-1, keepdim=True)
    if norm:
        r = dw - dot
        g = r / S
        eg = (edot + U * r.abs()) / S + r.abs() * eS / S ** 2 + U * g.abs()
    else:
        g, eg = dw, torch.zeros_like(dw)
    pgt = pj * g
    pg = pgt.sum(-1, keepdim=True)
    epg = (epj * g.abs() + pj * eg).sum(-1, keepdim=True) + k * U * pgt.abs().sum(-1, keepdim=True)
    G = torch.zeros_like(p).scatter(-1, ids, g)
    eG = torch.zeros_like(p).scatter(-1, ids, eg)
    d = G - pg
    ed = eG + epg + U * d.abs()
    dz = p * d
    err = (ep * d.abs() + p * ed + U * dz.abs()) * SECOND_ORDER
    return dz, err + half_ulp(dz, err, out_dtype)


# ---------------------------------------------------------------------------------------------------------------------
# index build and row-mover emulations
# ---------------------------------------------------------------------------------------------------------------------
def index_oracle(ids, E, rows):
    """Expected (counts, offsets, tile_expert[:tiles], num_m_tiles, pos, row_src) from ``_sorted_layout``."""
    from torchacc_b200.ops.moe import _sorted_layout
    flat = ids.reshape(-1)
    pos, off = _sorted_layout(ids, E)
    ok = (flat >= 0) & (flat < E)
    counts = torch.bincount(flat[ok], minlength=E)
    offsets = torch.tensor(off, dtype=I64, device=ids.device)
    tiles = off[-1] // TILE
    tile_expert = torch.repeat_interleave(torch.arange(E, device=ids.device), (offsets[1:] - offsets[:-1]) // TILE)
    row_src = torch.full((rows,), -1, dtype=I64, device=ids.device)
    row_src[pos[pos >= 0]] = (pos >= 0).nonzero().flatten()
    return counts, offsets, tile_expert, tiles, pos, row_src


def check_index(got, ids, E, rows, what):
    counts, offsets, tile_expert, tiles, pos, row_src = index_oracle(ids, E, rows)
    g_counts, g_offsets, g_te, g_tiles, g_pos, g_src = got
    expect_equal(g_counts.long(), counts, f"{what}: counts")
    expect_equal(g_offsets.long(), offsets, f"{what}: offsets")
    assert int(g_tiles) == tiles, f"{what}: num_m_tiles {int(g_tiles)} != {tiles}"
    expect_equal(g_te[:tiles].long(), tile_expert, f"{what}: tile_expert")
    expect_equal(g_pos.reshape(-1).long(), pos, f"{what}: pos")
    expect_equal(g_src.long(), row_src, f"{what}: row_src")


def emulate_permute(x, row_src, offsets, k, out):
    """x_perm[r] = x[row_src[r] // k] (zero on padding rows) for r < offsets[E]; rows past it untouched."""
    used = int(offsets[-1])
    src = row_src[:used].long()
    rows = x[src.clamp(min=0) // k].clone()
    rows[src < 0] = 0
    out[:used] = rows


def check_permute(x_perm, x, row_src, offsets, k, what):
    used = int(offsets[-1])
    src = row_src[:used].long()
    want = x[src.clamp(min=0) // k]
    want = torch.where((src < 0)[:, None], torch.zeros_like(want), want)
    expect_equal(bits(x_perm[:used]), bits(want), f"{what}: permuted rows")


def emulate_unpermute_sum(dx_perm, pos):
    """dx[t] = sum_j dx_perm[pos[t, j]] in fp32, j ascending, sentinels skipped; one rounding."""
    T, k = pos.shape
    acc = torch.zeros(T, dx_perm.shape[1], dtype=FP32, device=dx_perm.device)
    for j in range(k):
        p = pos[:, j].long()
        acc += torch.where((p >= 0)[:, None], dx_perm[p.clamp(min=0)].float(), torch.zeros_like(acc))
    return acc.to(dx_perm.dtype)


def emulate_combine_fwd(y_perm, pos, w, residual, fault=None):
    """out[t] = sum_j w[t, j] y_perm[pos[t, j]] (fp32 fma chain, j ascending) + residual[t], one rounding.  The exact
    tests use data on which every step is exact, so fp64 arithmetic rounded to fp32 per step emulates the fma."""
    T, k = pos.shape
    acc = torch.zeros(T, y_perm.shape[1], dtype=F64, device=y_perm.device)
    for j in range(k):
        p = pos[:, j].long()
        wj = w[:, j].float()
        if fault == "weights_16bit":
            wj = wj.to(y_perm.dtype).float()
        y = torch.where((p >= 0)[:, None], y_perm[p.clamp(min=0)].double(), torch.zeros_like(acc))
        acc = (acc + wj.double()[:, None] * y).float().double()
        if fault == "residual_in_loop" and residual is not None:
            acc = (acc + residual.double()).float().double()
    if fault == "residual_before_rounding":   # the weighted sum rounded to 16 bits first, then the residual added
        acc = acc.to(y_perm.dtype).double()
    if residual is not None and fault != "residual_in_loop":
        acc = acc + residual.double()
    return acc.float().to(y_perm.dtype)


def combine_ref(y_perm, pos, w, residual):
    """fp64 out[t] and, per element, sum over the fma chain of |partial sums| (the rounding-error weight)."""
    T, k = pos.shape
    acc = torch.zeros(T, y_perm.shape[1], dtype=F64, device=y_perm.device)
    weight = torch.zeros_like(acc)
    for j in range(k):
        p = pos[:, j].long()
        y = torch.where((p >= 0)[:, None], y_perm[p.clamp(min=0)].double(), torch.zeros_like(acc))
        acc = acc + (w[:, j].double()[:, None] if w is not None else 1.0) * y
        weight += acc.abs()
    if residual is not None:
        acc = acc + residual.double()
        weight += acc.abs()
    return acc, weight


def combine_bwd_ref(dout, y_perm, row_src, offsets, w, k):
    """(dy_perm as the kernel rounds it: fp32(w dout) then 16 bits, dy64, dw64 per used row, dw bound per used row).
    dw = <y, dout> reduced in a fixed order: each thread's fmaf chain over 8 elements per 16-byte vector and
    ceil(H / 2048) passes, 5 butterfly levels, then the 8 warps' partials added serially: every product passes
    through at most 8 ceil(H / 2048) + 5 + 8 roundings, so |err| <= that many u times sum |y_i dout_i|."""
    used = int(offsets[-1])
    src = row_src[:used].long()
    ok = src >= 0
    s = src.clamp(min=0)
    g = dout[s // k]
    ws = w.reshape(-1)[s].float()
    dy = (ws[:, None] * g.float()).to(dout.dtype)
    dy = torch.where(ok[:, None], dy, torch.zeros_like(dy))
    dy64 = torch.where(ok[:, None], ws.double()[:, None] * g.double(), torch.zeros_like(g, dtype=F64))
    prod = y_perm[:used].double() * g.double()
    dw64 = prod.sum(1)
    H = dout.shape[1]
    n = 8 * -(-H // (8 * 256)) + 5 + 8
    return dy, dy64, dw64, n * U * prod.abs().sum(1) * SECOND_ORDER, src, ok


# ---------------------------------------------------------------------------------------------------------------------
# MX-FP8 oracle: never uses torch's float8 cast
# ---------------------------------------------------------------------------------------------------------------------
def e4m3_values():
    """fp64 value of each of the 256 e4m3fn codes (NaN for 0x7f and 0xff)."""
    vals = []
    for c in range(256):
        s, e, m = c >> 7, (c >> 3) & 15, c & 7
        if e == 15 and m == 7:
            v = float("nan")
        elif e == 0:
            v = m / 8 * 2.0 ** -6
        else:
            v = (1 + m / 8) * 2.0 ** (e - 7)
        vals.append(-v if s else v)
    return torch.tensor(vals, dtype=F64)


_E4M3_POS = e4m3_values()[:127]    # codes 0..126: 0 .. 448, increasing


def e4m3_round(x):
    """Codes (uint8) of fp64 x rounded to nearest-even e4m3, saturating at +-448 and keeping the sign of zero (and of
    values that round to zero); NaN -> 0x7f."""
    table = _E4M3_POS.to(x.device)
    a = x.abs()
    hi = torch.searchsorted(table, a.clamp(max=448.0)).clamp(max=126)      # first code with value >= |x|
    lo = (hi - 1).clamp(min=0)
    dlo, dhi = a - table[lo], table[hi] - a
    code = torch.where(dlo < dhi, lo, hi)
    code = torch.where(dlo == dhi, torch.where(lo % 2 == 0, lo, hi), code)   # tie: the even code
    code = torch.where(a >= 448.0, torch.full_like(code, 126), code)
    code = code | (torch.signbit(x).long() << 7)
    code = torch.where(torch.isnan(x), torch.full_like(code, 0x7F), code)
    return code.to(U8)


def _scale_byte_table():
    """UE8M0 byte for every positive bf16 amax bit pattern (index = bits, 0..0x7f80): the smallest e >= 1 with
    2^(e - 127) >= amax / 448, by integer arithmetic; 254 for +inf (the kernel's clamp), 0 for amax = 0."""
    out = [0] * 0x7F81
    for b in range(1, 0x7F80):
        eb, mb = b >> 7, b & 127
        n, p = (128 + mb, eb - 134) if eb else (mb, -133)          # amax = n 2^p
        d = -12                                                    # smallest d with 7 2^d >= n: amax <= 448 2^(d+p-7)
        while (7 << d if d >= 0 else 7 / (1 << -d)) < n:
            d += 1
        out[b] = min(254, max(1, d + p + 121))                     # 448 2^(e - 127) = 7 2^(e - 121)
    out[0x7F80] = 254
    return torch.tensor(out, dtype=torch.int64)


_SCALE_TABLE = None


def scale_bytes(amax_bf16):
    global _SCALE_TABLE
    if _SCALE_TABLE is None:
        _SCALE_TABLE = _scale_byte_table()
    b = bits(amax_bf16.contiguous()).long() & 0x7FFF
    return _SCALE_TABLE.to(amax_bf16.device)[b]


def pow2(n):
    """2^n in fp64 for integer tensors n in [-1022, 1023], built from the exponent bits (torch.pow on the GPU is not
    exact for every n)."""
    return ((n.long() + 1023) << 52).view(F64)


def mx_oracle(x):
    """(codes [R, C] uint8, scale matrix [R, ceil(C / 32)] int64) of bf16 x quantised along C as the kernel does it:
    amax ignores NaN (fmaxf); an infinite amax clamps the byte at 254, and the kernel's inverse scale for byte 254 is
    the fp32 bit pattern (254 - 254) << 23 = 0, so the finite elements of such a block become +-0 and the infinity
    NaN."""
    R, C = x.shape
    Cp = -(-C // 32) * 32
    xp = torch.zeros(R, Cp, dtype=BF16, device=x.device)
    xp[:, :C] = x
    blk = xp.view(R, Cp // 32, 32)
    a = blk.abs()
    amax = torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(-1)
    e = scale_bytes(amax)
    inv = torch.where(e == 254, torch.zeros_like(e, dtype=F64), pow2(127 - e))
    v = blk.double() * inv[..., None]
    codes = e4m3_round(v).view(R, Cp)[:, :C]
    return codes, e


def atoms(scales, R, K):
    """Scale matrix [R, K / 32] (K in elements) -> the atom-tiled byte layout of csrc/ops/quant_mxfp8.cu, with the
    padding of the last row and K atoms zero."""
    ar, ak = -(-R // 128), -(-K // 128)
    full = torch.zeros(ar * 128, ak * 4, dtype=U8, device=scales.device)
    full[:R, :scales.shape[1]] = scales.to(U8)
    return full.view(ar, 4, 32, ak, 4).permute(0, 3, 2, 1, 4).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers: the C ABI called directly
# ---------------------------------------------------------------------------------------------------------------------
def _nat():
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import fp8, moe  # noqa: F401  (register the signatures)
    return nat, nat.require()


_DT = {FP32: 0, BF16: 1, FP16: 2}


def router_fwd(logits, k, norm):
    nat, L = _nat()
    T, E = logits.shape
    w = Guarded((T, k), FP32)
    ids = Guarded((T, k), I64)
    nat.check(L.tb_moe_router_fwd(logits.data_ptr(), w.view.data_ptr(), ids.view.data_ptr(), T, E, k, int(norm),
                                  _DT[logits.dtype], nat.stream()), "tb_moe_router_fwd")
    return w, ids


def router_bwd(logits, ids, dw, norm):
    nat, L = _nat()
    T, E = logits.shape
    dl = Guarded((T, E), logits.dtype)
    nat.check(L.tb_moe_router_bwd(logits.data_ptr(), ids.data_ptr(), dw.data_ptr(), dl.view.data_ptr(), T, E,
                                  ids.shape[1], int(norm), _DT[logits.dtype], nat.stream()), "tb_moe_router_bwd")
    return dl


def index_build(ids, E):
    """tb_moe_index with every output guarded; returns (rows, guarded outputs)."""
    from torchacc_b200.ops.moe import capacity
    nat, L = _nat()
    T, k = ids.shape
    rows = capacity(T, k, E)
    outs = [Guarded((E,), I32), Guarded((E + 1,), I32), Guarded((rows // TILE,), I32), Guarded((1,), I32),
            Guarded((T, k), I32), Guarded((rows,), I32)]
    nat.check(L.tb_moe_index(ids.data_ptr(), T, k, E, rows, *[g.view.data_ptr() for g in outs], nat.stream()),
              "tb_moe_index")
    return rows, outs


# ---------------------------------------------------------------------------------------------------------------------
# 1. router
# ---------------------------------------------------------------------------------------------------------------------
EK = [(1, 1)] + [(E, k) for E in (8, 60, 64, 128, 256) for k in (1, 2, 4, 8) if k <= E]
T_S = [1, 7, 8, 9, 8192]


def router_logits(pattern, T, E, dtype, gen):
    if pattern == "gaussian":   # on multiples of 2^-8 (exact in fp16, coarser in bf16): distinct values stay apart
        return (torch.round(torch.randn(T, E, generator=gen, device=DEV) * 512) / 256).to(dtype)
    if pattern == "ties":                                          # many experts on the same bf16 value
        return torch.randint(-3, 4, (T, E), generator=gen, device=DEV).to(dtype) * 0.5
    if pattern == "peaked":                                        # one expert >= 110 above the rest
        z = torch.randint(-8, 8, (T, E), generator=gen, device=DEV).to(FP32) * 0.25
        hot = torch.randint(0, E, (T,), generator=gen, device=DEV)
        z[torch.arange(T, device=DEV), hot] = 112.0
        return z.to(dtype)
    raise ValueError(pattern)


def _router_case(logits, k, norm, gen, what, used):
    T, E = logits.shape
    z = logits.double()
    p, want = router_oracle(logits, k)
    router_premise(p, k, what)
    w, ids = router_fwd(logits, k, norm)
    dw = torch.randn(T, k, generator=gen, device=DEV)
    dl = router_bwd(logits, ids.view, dw, norm)
    torch.cuda.synchronize()
    w.check_untouched(f"{what}: weights")
    ids.check_untouched(f"{what}: ids")
    dl.check_untouched(f"{what}: d(logits)")
    expect_equal(ids.view, want, f"{what}: ids")
    w64, wb = router_weights_bound(z, p, want, norm)
    used["w"] = max(used.get("w", 0), within(w.view, w64, wb, f"{what}: weights"))
    dz, db = router_dlogits_bound(z, p, want, dw, norm, logits.dtype)
    used["dz"] = max(used.get("dz", 0), within(dl.view, dz, db, f"{what}: d(logits)"))


@gpu
@pytest.mark.parametrize("pattern", ["gaussian", "ties", "peaked"])
@pytest.mark.parametrize("dtype", [FP32, BF16, FP16], ids=["fp32", "bf16", "fp16"])
def test_router(dtype, pattern):
    """Every valid (E, k) of E in {1, 8, 60, 64, 128, 256} x k in {1, 2, 4, 8}, norm on and off, T in {1, 7, 8, 9,
    8192} (8 tokens per CTA): ids exact, weights and d(logits) within the derived bounds."""
    gen = torch.Generator(device=DEV).manual_seed(11)
    used = {}
    for E, k in EK:
        for T in T_S:
            logits = padded_input(router_logits(pattern, T, E, dtype, gen))
            for norm in (False, True):
                _router_case(logits, k, norm, gen, f"{pattern} {dtype} E={E} k={k} T={T} norm={norm}", used)
    print(f"[bound] router {dtype} {pattern}: largest fraction used {used}")


@gpu
def test_router_3d_input_and_autograd_entry():
    """``moe_router`` on a [B, S, E] bf16 input: the same ids, weights and d(logits) as the flat kernel calls."""
    from torchacc_b200.ops.moe import moe_router
    gen = torch.Generator(device=DEV).manual_seed(12)
    z = router_logits("gaussian", 3 * 37, 60, BF16, gen).view(3, 37, 60).requires_grad_(True)
    w, ids = moe_router(z, 4, True)
    g = torch.randn(w.shape, generator=gen, device=DEV)
    w.backward(g)
    wf, idf = router_fwd(z.detach().reshape(-1, 60), 4, True)
    dl = router_bwd(z.detach().reshape(-1, 60), idf.view, g.reshape(-1, 4).contiguous(), True)
    torch.cuda.synchronize()
    assert w.shape == (3, 37, 4) and ids.shape == (3, 37, 4)
    expect_equal(ids.reshape(-1, 4), idf.view, "3-D ids")
    expect_equal(w.detach().reshape(-1, 4), wf.view, "3-D weights")
    expect_equal(z.grad.reshape(-1, 60), dl.view, "3-D d(logits)")
    _router_case(z.detach().reshape(-1, 60), 4, True, gen, "3-D", {})


@gpu
@pytest.mark.parametrize("dtype", [FP32, BF16, FP16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("E,k", [(8, 2), (60, 4), (256, 8)])
def test_router_non_finite_rows(dtype, E, k):
    """Rows with a NaN, a +inf, all -inf or all NaN logits among normal rows: each picks k distinct experts in [0, E)
    (0..k-1: NaN ranks first, as in torch.topk) with NaN weights and NaN d(logits), and makes its ``moe_experts``
    output non-finite; every other row is bitwise what a run without the bad rows gives, forward and backward."""
    from torchacc_b200.ops.moe import moe_experts
    gen = torch.Generator(device=DEV).manual_seed(13)
    T = 40
    z = router_logits("gaussian", T, E, dtype, gen)
    inf = float("inf")
    bad = [3, 8, 9, 17, 31, 39]
    z[3, E // 2] = float("nan")
    z[8, E - 1] = inf
    z[9] = -inf
    z[17] = float("nan")
    z[31, 0] = inf
    z[31, 1] = -inf
    z[39, :E // 2] = -inf                                          # half -inf: still a normal row ...
    z[39, E // 2] = float("nan")                                   # ... until one NaN
    z[5, :E - 1] = -inf                                            # normal rows with -inf logits
    good = [t for t in range(T) if t not in bad]
    assert bool(bad_rows(z.double())[bad].all()) and not bool(bad_rows(z.double())[good].any())
    dw = torch.randn(T, k, generator=gen, device=DEV)
    for norm in (False, True):
        w, ids = router_fwd(z, k, norm)
        dl = router_bwd(z, ids.view, dw, norm)
        zc = z[good].contiguous()
        wc, idc = router_fwd(zc, k, norm)
        dlc = router_bwd(zc, idc.view, dw[good].contiguous(), norm)
        torch.cuda.synchronize()
        for g_ in (w, ids, dl):
            g_.check_untouched(f"non-finite rows norm={norm}")
        want = torch.arange(k, device=DEV).expand(len(bad), k)
        expect_equal(ids.view[bad], want, f"ids of the bad rows (norm={norm})")
        assert bool(torch.isnan(w.view[bad]).all()), "a bad row has a non-NaN weight"
        assert bool(torch.isnan(dl.view[bad]).all()), "a bad row has a non-NaN d(logit)"
        expect_equal(ids.view[good], idc.view, "ids of the other rows")
        expect_equal(w.view[good], wc.view, "weights of the other rows")
        expect_equal(dl.view[good], dlc.view, "d(logits) of the other rows")
    H, Fd = 64, 128
    x = torch.randn(T, H, generator=gen, device=DEV).to(BF16)
    wgu = (torch.randn(E, 2 * Fd, H, generator=gen, device=DEV) / 8).to(BF16)
    wd = (torch.randn(E, H, Fd, generator=gen, device=DEV) / 8).to(BF16)
    out = moe_experts(x, ids.view, w.view, wgu, wd)
    torch.cuda.synchronize()
    assert not bool(torch.isfinite(out[bad]).any()), "a bad row's output is finite: its token was dropped"
    assert bool(torch.isfinite(out[good]).all())


# ---------------------------------------------------------------------------------------------------------------------
# 2. index build
# ---------------------------------------------------------------------------------------------------------------------
def _index_case(ids, E, what):
    rows, outs = index_build(ids, E)
    torch.cuda.synchronize()
    for g_ in outs:
        g_.check_untouched(what)
    tiles = int(outs[3].view[0])
    outs[2].check_untouched(f"{what}: tile_expert past num_m_tiles",
                            torch.arange(rows // TILE, device=DEV) >= tiles)
    check_index([g_.view for g_ in outs[:3]] + [outs[3].view[0]] + [g_.view for g_ in outs[4:]], ids, E, rows, what)
    print(f"[exact] index {what}: n={ids.numel()} E={E} tiles={tiles}")


def straddle_ids(E, k, T, gen):
    """Random ids with experts 1, 2, 3 holding 127, 128 and 129 entries that straddle a 1024-entry round."""
    n = T * k
    flat = torch.randint(4, E, (n,), generator=gen, device=DEV)
    for e, c in ((1, 127), (2, 128), (3, 129)):
        start = e * ROUND - c // 2
        flat[start:start + c] = e
    return flat.view(T, k)


@gpu
@pytest.mark.parametrize("case", ["e256_k8_t8192", "n_mod_0", "n_mod_1", "n_mod_1023", "n_lt_32", "t0",
                                  "all_last_expert", "straddle", "out_of_range"])
def test_index_build(case):
    gen = torch.Generator(device=DEV).manual_seed(14)
    E, k, T = {"e256_k8_t8192": (256, 8, 8192), "n_mod_0": (60, 4, 512), "n_mod_1": (64, 1, 2049),
               "n_mod_1023": (8, 1, 3071), "n_lt_32": (8, 4, 5), "t0": (8, 2, 0), "all_last_expert": (64, 8, 300),
               "straddle": (16, 2, 2000), "out_of_range": (60, 4, 700)}[case]
    if case == "all_last_expert":
        ids = torch.full((T, k), E - 1, dtype=I64, device=DEV)
    elif case == "straddle":
        ids = straddle_ids(E, k, T, gen)
    else:
        ids = torch.randint(0, E, (T, k), generator=gen, device=DEV)
    if case == "out_of_range":   # all dropped: compared in 64 bits before narrowing
        bad = torch.tensor([-1, E, E + 1, 2 ** 31 - 1, 2 ** 32 + 3, 2 ** 32, -2 ** 32 + 1, -2 ** 32 + E - 1,
                            2 ** 63 - 1, -2 ** 63], device=DEV)
        where = torch.randperm(T * k, generator=gen, device=DEV)[:bad.numel() * 40]
        ids.view(-1)[where] = bad.repeat(40)
    _index_case(padded_input(ids, poison=2 ** 40), E, case)


# ---------------------------------------------------------------------------------------------------------------------
# 3. row movers
# ---------------------------------------------------------------------------------------------------------------------
def _mover_setup(dtype, k, H, T, E, gen, sentinels=True):
    ids = torch.rand(T, E, generator=gen, device=DEV).argsort(-1)[:, :k]
    if sentinels:
        ids[::5, k - 1] = E                                       # HF's "no expert" sentinel
        ids[::7, 0] = -1
    from torchacc_b200.ops.moe import MoEIndex
    idx = MoEIndex(ids, E)
    return ids, idx


def _ints(shape, lim, gen, dtype):
    return torch.randint(-lim, lim + 1, shape, generator=gen, device=DEV).to(dtype)


MOVER_GRID = [(dt, k, H) for dt in (BF16, FP16) for k in (1, 2, 8) for H in (8, 200, 2048, 4096)]


@gpu
@pytest.mark.parametrize("dtype,k,H", MOVER_GRID, ids=[f"{'bf16' if d == BF16 else 'fp16'}-k{k}-H{h}"
                                                       for d, k, h in MOVER_GRID])
def test_row_movers(dtype, k, H):
    """permute, unpermute-sum, combine forward and backward through the C ABI on 3 SMs (24 CTAs: every kernel
    grid-strides), with sentinel ids, canaries around every output and NaN around every input."""
    nat, L = _nat()
    gen = torch.Generator(device=DEV).manual_seed(15 + k + H)
    T, E = 300, 16
    ids, idx = _mover_setup(dtype, k, H, T, E, gen)
    rows, sms, bf = idx.rows, 3, int(dtype == BF16)
    offsets = idx.offsets.long()
    used = int(offsets[-1])
    what = f"{dtype} k={k} H={H}"
    # permute: a bitwise copy, zero padding rows, rows past offsets[E] untouched
    x = padded_input(torch.randn(T, H, generator=gen, device=DEV).to(dtype))
    xp = Guarded((rows, H), dtype)
    nat.check(L.tb_moe_permute(x.data_ptr(), idx.row_src.data_ptr(), idx.offsets.data_ptr(), xp.view.data_ptr(), rows,
                               k, E, H, sms, nat.stream()), "tb_moe_permute")
    # unpermute-sum, exact: small integers (|sum| <= 8 * 64)
    dxp = padded_input(_ints((rows, H), 64, gen, dtype))
    dx = Guarded((T, H), dtype)
    nat.check(L.tb_moe_unpermute_sum(dxp.data_ptr(), idx.pos.data_ptr(), dx.view.data_ptr(), T, k, H, sms,
                                     nat.stream(), bf), "tb_moe_unpermute_sum")
    # combine forward, exact: integers |y| <= 64 times weights that are multiples of 2^-12 in [-1, 1], plus an integer
    # residual |r| <= 1000: every partial sum is a multiple of 2^-12 below 2^11, so 23 bits hold it exactly
    assert 8 * 64 + 1000 < 2 ** 11 and k <= 8
    yp = padded_input(_ints((rows, H), 64, gen, dtype))
    w = padded_input(torch.randint(-4096, 4097, (T, k), generator=gen, device=DEV).float() / 4096)
    res = padded_input(_ints((T, H), 1000, gen, dtype))
    out = Guarded((T, H), dtype)
    nat.check(L.tb_moe_combine_fwd(yp.data_ptr(), idx.pos.data_ptr(), w.data_ptr(), res.data_ptr(), out.view.data_ptr(),
                                   T, k, H, sms, nat.stream(), bf), "tb_moe_combine_fwd")
    out_nr = Guarded((T, H), dtype)
    nat.check(L.tb_moe_combine_fwd(yp.data_ptr(), idx.pos.data_ptr(), w.data_ptr(), 0, out_nr.view.data_ptr(),
                                   T, k, H, sms, nat.stream(), bf), "tb_moe_combine_fwd")
    # combine backward: Gaussian dout, y_perm and weights
    dout = padded_input(torch.randn(T, H, generator=gen, device=DEV).to(dtype))
    ypg = padded_input(torch.randn(rows, H, generator=gen, device=DEV).to(dtype))
    wg = padded_input(torch.rand(T, k, generator=gen, device=DEV))
    dyp = Guarded((rows, H), dtype)
    dwg = Guarded((T, k), FP32)
    nat.check(L.tb_moe_combine_bwd(dout.data_ptr(), ypg.data_ptr(), idx.row_src.data_ptr(), idx.offsets.data_ptr(),
                                   wg.data_ptr(), dyp.view.data_ptr(), dwg.view.data_ptr(), rows, k, E, H, sms,
                                   nat.stream(), bf), "tb_moe_combine_bwd")
    torch.cuda.synchronize()
    past = (torch.arange(rows, device=DEV) >= used)[:, None].expand(rows, H)
    xp.check_untouched(f"permute {what}", past)
    check_permute(xp.view, x, idx.row_src, offsets, k, f"permute {what}")
    dx.check_untouched(f"unpermute {what}")
    ref, _ = combine_ref(dxp, idx.pos, None, None)
    expect_rounded(dx.view, ref, f"unpermute-sum {what}")
    for o, r in ((out, res), (out_nr, None)):
        o.check_untouched(f"combine fwd {what}")
        ref, _ = combine_ref(yp, idx.pos, w, r)
        expect_rounded(o.view, ref, f"combine fwd {what} residual={r is not None}")
    dy, dy64, dw64, dwb, src, ok = combine_bwd_ref(dout, ypg, idx.row_src, offsets, wg, k)
    dyp.check_untouched(f"combine bwd {what}", past)
    expect_equal(bits(dyp.view[:used]), bits(dy), f"combine bwd d(y_perm) {what}: fp32(w dout) then 16 bits")
    within(dyp.view[:used], dy64, ulp_dtype(dy64, dtype), f"combine bwd d(y_perm) {what}: 1 ulp of fp64")
    sent = (idx.pos < 0)
    dwg.check_untouched(f"combine bwd dw {what}: sentinel entries", sent)
    within(dwg.view.reshape(-1)[src[ok]], dw64[ok], dwb[ok] + 2.0 ** -149, f"combine bwd dw {what}")
    print(f"[exact] row movers {what}: rows={rows} used={used}")


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("k", [1, 2, 8])
def test_combine_and_unpermute_gaussian(dtype, k):
    """Gaussian data on every SM: unpermute-sum within (k - 1) fp32 roundings plus half an ulp, combine forward within
    its k fma roundings plus the residual's add plus half an ulp (both weighted by the partial sums they round)."""
    nat, L = _nat()
    gen = torch.Generator(device=DEV).manual_seed(16 + k)
    T, E, H = 2000, 16, 512
    ids, idx = _mover_setup(dtype, k, H, T, E, gen)
    bf = int(dtype == BF16)
    dxp = torch.randn(idx.rows, H, generator=gen, device=DEV).to(dtype)
    w = torch.rand(T, k, generator=gen, device=DEV)
    res = torch.randn(T, H, generator=gen, device=DEV).to(dtype)
    dx = Guarded((T, H), dtype)
    out = Guarded((T, H), dtype)
    nat.check(L.tb_moe_unpermute_sum(dxp.data_ptr(), idx.pos.data_ptr(), dx.view.data_ptr(), T, k, H, nat.num_sms(),
                                     nat.stream(), bf), "tb_moe_unpermute_sum")
    nat.check(L.tb_moe_combine_fwd(dxp.data_ptr(), idx.pos.data_ptr(), w.data_ptr(), res.data_ptr(), out.view.data_ptr(),
                                   T, k, H, nat.num_sms(), nat.stream(), bf), "tb_moe_combine_fwd")
    torch.cuda.synchronize()
    dx.check_untouched("unpermute")
    out.check_untouched("combine")
    ref, wt = combine_ref(dxp, idx.pos, None, None)
    err = U * wt * SECOND_ORDER                         # one rounding per partial sum
    within(dx.view, ref, err + half_ulp(ref, err, dtype), f"unpermute-sum gaussian {dtype} k={k}")
    ref, wt = combine_ref(dxp, idx.pos, w, res)
    err = U * wt * SECOND_ORDER
    within(out.view, ref, err + half_ulp(ref, err, dtype), f"combine fwd gaussian {dtype} k={k}")


@gpu
@pytest.mark.parametrize("fp8_path", [False, True], ids=["bf16", "fp8"])
def test_moe_mlp_empty_batch(fp8_path):
    """``MoEMLP`` on T = 0 tokens: an empty output, and zero weight gradients."""
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops.moe import MoEMLP
    torch.manual_seed(0)
    with torch.device(DEV):
        mlp = MoEMLP(256, 256, 8, 2, dtype=BF16)
    for p in mlp.parameters():
        torch.nn.init.normal_(p, 0, 0.05)
    prev = fp8.enabled()
    fp8.enable(fp8_path)
    try:
        x = torch.zeros(0, 256, device=DEV, dtype=BF16, requires_grad=True)
        out = mlp(x, residual=x)
        out.float().sum().backward()
    finally:
        fp8.enable(prev)
    torch.cuda.synchronize()
    assert out.shape == (0, 256)
    for n, p in mlp.named_parameters():
        assert p.grad is not None and bool((p.grad == 0).all()), n


# ---------------------------------------------------------------------------------------------------------------------
# 4. MX-FP8 quantiser
# ---------------------------------------------------------------------------------------------------------------------
def quant(x, ldq=None, ldqt=None, rowwise=True, colwise=True):
    """tb_quant_mxfp8 on x (any row pitch) into guarded payloads with pitches ldq / ldqt and guarded scale buffers."""
    nat, L = _nat()
    R, C = x.shape
    ldq = ldq or -(-C // 16) * 16
    ldqt = ldqt or -(-R // 16) * 16
    n_sf = -(-R // 128) * -(-C // 128) * 512
    q = Guarded((R, ldq), U8) if rowwise else None
    qt = Guarded((C, ldqt), U8) if colwise else None
    sf = Guarded((n_sf,), U8) if rowwise else None
    sft = Guarded((n_sf,), U8) if colwise else None
    p = lambda g: 0 if g is None else g.view.data_ptr()   # noqa: E731
    code = L.tb_quant_mxfp8(x.data_ptr(), x.stride(0), R, C, p(q), ldq, p(sf), p(qt), ldqt, p(sft), nat.stream())
    nat.check(code, "tb_quant_mxfp8")
    return q, sf, qt, sft


def _nan_code(c):
    return (c & 0x7F) == 0x7F


def check_quant(x, outs, what):
    """Payload and scale bytes of both orientations against the oracle; pitch gaps and pads untouched."""
    R, C = x.shape
    q, sf, qt, sft = outs
    for g_, xx, n, k, name in ((q, x, R, C, "row-wise"), (qt, x.t(), C, R, "transposed")):
        s_g = sf if g_ is q else sft
        codes, scales = mx_oracle(xx.contiguous())
        gap = torch.zeros_like(g_.view, dtype=torch.bool)
        gap[:, k:] = True
        g_.check_untouched(f"{what} {name}: payload pitch gap", gap)
        s_g.check_untouched(f"{what} {name}: scales")
        got = g_.view[:, :k]
        nan_ok = _nan_code(codes) & _nan_code(got)
        bad = (got != codes) & ~nan_ok
        if bool(bad.any()):
            i, j = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what} {name}: {int(bad.sum())} payload bytes differ; first at {[i, j]}: x "
                                 f"{xx[i, j].item()!r} (block {xx[i, j // 32 * 32:j // 32 * 32 + 32].tolist()}) byte "
                                 f"{int(got[i, j]):#x} want {int(codes[i, j]):#x}, scale byte "
                                 f"{int(scales[i, j // 32])}")
        expect_equal(s_g.view, atoms(scales, n, k), f"{what} {name}: scale bytes (atom layout)")


def _amax_levels():
    """bf16 amax values (as fp32): the ends and middle of the scale range, the bf16 subnormals, and 448 2^j with one
    bf16 ulp either side of it."""
    def bf(b):
        return torch.tensor([b], dtype=torch.int16).view(BF16).float().item()
    lv = [bf(1), bf(2), bf(0x3F), bf(0x7F), bf(0x80), bf(0x81), 1.0, 3.0, 448.0, bf(0x7F7F), bf(0x7F7E)]
    for j in (-133, -120, -100, -20, -1, 0, 1, 20, 100, 119):
        v = torch.tensor([448.0 * 2.0 ** j], dtype=F64)
        if v.item() < 3.3e38 and v.item() > 9.2e-41:
            b = int(bits(v.float().to(BF16)))
            lv += [bf(b - 1), bf(b), bf(b + 1)]
    return sorted(set(x for x in lv if 0 < x < 3.4e38))


@gpu
def test_quant_exhaustive_bf16():
    """Every finite bf16 bit pattern as an element, under each amax level of ``_amax_levels`` that bounds it: each
    32-element block holds its level (with a random sign) and 31 patterns no larger.  Payload and scale bytes of both
    orientations from one call, exact."""
    allb = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    vals = allb.view(BF16)
    vals = vals[torch.isfinite(vals.float())]
    rows = []
    g = torch.Generator().manual_seed(17)
    for a in _amax_levels():
        pool = vals[vals.float().abs() <= a]
        pool = pool[torch.randperm(pool.numel(), generator=g)]
        nb = -(-pool.numel() // 31)
        pool = pool.repeat(-(-nb * 31 // pool.numel()))[:nb * 31].view(nb, 31)
        lead = torch.full((nb, 1), a, dtype=F64)
        lead = torch.where(torch.rand(nb, 1, generator=g) < 0.5, -lead, lead).to(BF16)
        blk = torch.cat([lead, pool], 1)
        perm = torch.argsort(torch.rand(nb, 32, generator=g), 1)
        rows.append(torch.gather(blk, 1, perm))
    blocks = torch.cat(rows)                                   # [n, 32]
    n = blocks.shape[0] // 12 * 12
    x = blocks[:n].reshape(-1, 384).to(DEV)                    # 12 blocks per row
    q = quant(x)
    torch.cuda.synchronize()
    check_quant(x, q, "exhaustive")
    print(f"[exact] quantiser: {x.numel()} elements, {len(_amax_levels())} amax levels")


SHAPES = [1, 31, 33, 128, 129, 200, 384]


@gpu
@pytest.mark.parametrize("R", SHAPES)
def test_quant_shapes_and_pitches(R):
    """R x C for C in the same set, with the input's row pitch and both payload pitches wider than the rows; the
    padding of the last atoms must be written as zero bytes and nothing else outside the views."""
    gen = torch.Generator(device=DEV).manual_seed(18 + R)
    for C in SHAPES:
        ldx = -(-C // 8) * 8 + 24
        buf = torch.full((R + 2, ldx), float("nan"), dtype=BF16, device=DEV)
        x = buf[1:R + 1, :C]
        scale = torch.exp2(torch.randint(-20, 20, (R, 1), generator=gen, device=DEV).float())
        x.copy_((torch.randn(R, C, generator=gen, device=DEV) * scale).to(BF16))
        q = quant(x, ldq=-(-C // 16) * 16 + 32, ldqt=-(-R // 16) * 16 + 16)
        torch.cuda.synchronize()
        check_quant(x, q, f"R={R} C={C}")


@gpu
def test_quant_non_finite_and_reference():
    """A NaN element leaves its block's scale to the finite elements and quantises to NaN alone; an infinite element
    clamps the scale byte at 254 and turns its block's finite elements into +-0 and itself into NaN; an all-NaN block
    has scale byte 0.  ``quantize_mxfp8_ref`` gives the same values, and an MX-FP8 GEMM fed such blocks returns
    non-finite values exactly in the rows and columns they touch."""
    from torchacc_b200.ops import fp8
    gen = torch.Generator(device=DEV).manual_seed(19)
    M, N, K = 256, 256, 256
    a = torch.randn(M, K, generator=gen, device=DEV).to(BF16)
    b = torch.randn(N, K, generator=gen, device=DEV).to(BF16)
    nan, inf = float("nan"), float("inf")
    a[3, 40] = nan
    a[7, 100] = inf
    a[9, 200] = -inf
    a[11, 64:96] = nan
    b[5, 130] = nan
    b[200, 0] = -inf
    for x in (a, b):
        check_quant(x, quant(x), "non-finite")
    ar, _ = fp8.quantize_mxfp8(a)
    br, _ = fp8.quantize_mxfp8(b)
    for t, x in ((ar, a), (br, b)):
        expect_equal(fp8.dequantize_mxfp8(t), fp8.quantize_mxfp8_ref(x), "quantize_mxfp8_ref on non-finite blocks")
    blk = fp8.dequantize_mxfp8(ar)
    assert bool(torch.isnan(blk[7, 100])) and bool((blk[7, 96:100] == 0).all()) and bool(torch.isnan(blk[11, 64:96]).all())
    assert float(blk[3, 41]) != 0.0 and bool(torch.isnan(blk[3, 40]))
    d = fp8.gemm_mxfp8(ar, br)
    torch.cuda.synchronize()
    rows = torch.zeros(M, dtype=torch.bool, device=DEV)
    rows[[3, 7, 9, 11]] = True
    cols = torch.zeros(N, dtype=torch.bool, device=DEV)
    cols[[5, 200]] = True
    touched = rows[:, None] | cols[None, :]
    assert not bool(torch.isfinite(d[touched]).any()), "a row or column with a non-finite block has a finite output"
    assert bool(torch.isfinite(d[~touched]).all())


@gpu
def test_quant_rejects_misaligned_base_and_linear_copies_it():
    """``tb_quant_mxfp8`` refuses an input or payload base that is not 16-byte aligned (cudaErrorInvalidValue) without
    launching; ``linear()`` under fp8 on a view 2 bytes into its storage gives bitwise the result of an aligned copy,
    forward and backward."""
    from torchacc_b200.ops import fp8
    from torchacc_b200.ops.linear import linear
    nat, L = _nat()
    T, K, N = 256, 256, 384
    x0 = torch.randn(T * K + 8, device=DEV).to(BF16)
    xm = x0[1:1 + T * K].view(T, K)
    assert xm.data_ptr() % 16 == 2
    q = torch.empty(T, K, dtype=U8, device=DEV)
    sf = torch.zeros(2 * 2 * 512, dtype=U8, device=DEV)
    assert L.tb_quant_mxfp8(xm.data_ptr(), K, T, K, q.data_ptr(), K, sf.data_ptr(), 0, 0, 0, nat.stream()) == 1
    qm = torch.empty(T * K + 16, dtype=U8, device=DEV)[1:1 + T * K]
    xa = xm.clone()
    assert L.tb_quant_mxfp8(xa.data_ptr(), K, T, K, qm.data_ptr(), K, sf.data_ptr(), 0, 0, 0, nat.stream()) == 1
    torch.cuda.synchronize()
    w = (torch.randn(N, K, device=DEV) / 16).to(BF16)
    g = torch.randn(T, N, device=DEV).to(BF16)
    assert fp8.eligible(xm, w)
    prev = fp8.enabled()
    fp8.enable(True)
    try:
        results = []
        for xin in (xm, xa):
            xl = xin.detach().requires_grad_(True)
            wl = w.clone().requires_grad_(True)
            y = linear(xl, wl)
            y.backward(g)
            results.append((y.detach(), xl.grad, wl.grad))
    finally:
        fp8.enable(prev)
    torch.cuda.synchronize()
    for name, a_, b_ in zip(("y", "dx", "dw"), *results):
        expect_equal(a_, b_, f"fp8 linear on a 2-byte offset view: {name}")
    assert results[0][0].dtype == BF16 and bool(torch.isfinite(results[0][0]).all())
