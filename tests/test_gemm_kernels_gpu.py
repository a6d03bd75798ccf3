"""The GEMM kernels (csrc/gemm/gemm_bf16.cu: dense, SwiGLU, grouped; csrc/gemm/gemm_mxfp8.cu) against fp64 references,
bit for bit where the arithmetic allows it.

Premise of the exact tests.  The operands are small integers (times a power of two for MX-FP8).  Every product of two
16-bit integers is exact, and while every partial sum stays below 2^24 in magnitude it is an integer that fp32 holds
exactly, in whatever order and grouping the tensor cores add the products.  So the fp32 accumulator equals the fp64
reference exactly, bias and addend (integers too) are added in fp32 without error, and the only rounding left is the
epilogue's cast: the output must equal ``ref64.to(float32).to(out_dtype)`` exactly (compared with ``==``; a NaN fails).
Each test asserts the 2^24 bound on its inputs.  Magnitudes are chosen so that 16-bit outputs are mostly inexact and
often exact ties, which pins round-to-nearest-even.  The MX-FP8 kernel adds the 32 products of a scale block in a
datapath with about 13 fraction bits: its tests keep each block sum a sum of at most 32 integers of at most 7 bits
(|q| <= 8 per factor, one power of two per block), which that datapath holds exactly, and the scaled block sums again
below 2^24.  This premise held on an H100 for every test below.

Coverage of the dense kernel (``test_dense_exact``).  The kernel is instantiated per dtype (bf16, fp16), operand majors
(4) and epilogue path (staged: 16-byte aligned D; register: D one element off), 16 instantiations; the epilogue
variant (8) and the shape are runtime arguments.  Each instantiation j runs 8 cases i = 0..7 with epilogue E[i],
N = N_S[(i + 3j) % 8], M = M_S[(i + j) % 6], K = K_S[(i + 2j) % 7] and the schedule (static, dynamic)[(i + j) % 2].
For fixed j the maps i -> E[i] and i -> N index are bijections on 8 values, and 8 consecutive i cover all 6 M and all
7 K residues, so every instantiation meets every epilogue, every M in {1, 77, 128, 129, 1000, 1100} (1100: a full
raster group of 8 row tiles followed by a group of one), every N in {1, 3, 7, 13, 255, 256, 257, 520} (N < 8, the
scalar tail of ``store_row8``, 1 past a tile) and every K in {8, 16, 56, 64, 72, 100, 136} (K % 8 != 0 with a wider
pitch, K < 64, 1 past a K block), under both schedules; the offsets 3j and 2j vary the pairings across instantiations.
The staged path also needs D's rows to end on a 16-byte boundary (N % 8 == 0 for 16-bit, N % 4 == 0 for fp32): with
the other N the "staged" instantiations check that such outputs take the register path and keep their canaries, and a
second pass of 8 cases runs every epilogue once more at N in {256, 520, 136} (i -> E[i] again a bijection, M, K and the
schedule offset), where the staged kernel does run.  An fp32 addend that is not D always takes the register path (the
host stages fp32 only as a reduce-add into D).

Canaries.  Every output is a view inside a buffer of sentinel NaN bits: elements before the base, a pitch gap after
every row and spare rows after the last must keep those bits.  Every input sits inside a NaN-filled buffer (pitch gap,
two rows before and after), so a read past M, N or K poisons the output where the tensor map's extent zero-fills.

Bounds for non-integer data (the SwiGLU activation, Gaussian operands) are in ulps of the output dtype plus a floor
derived from the fp32 arithmetic next to each check, printed as ``[ulp]`` lines with the fraction of the bound used.

The tests without the ``gpu`` mark run the same checkers on a PyTorch emulation of the kernel's tile loop with planted
faults, and must reject every one of them."""
import pytest
import torch

gpu = pytest.mark.gpu
DEV = "cuda"
BF16, FP16, FP32 = torch.bfloat16, torch.float16, torch.float32
TILE_M, TILE_N, GROUP_M = 128, 256, 8
EXACT_LIMIT = 2.0 ** 24


# ---------------------------------------------------------------------------------------------------------------------
# checkers (device agnostic: the CPU tests below run them on an emulated kernel)
# ---------------------------------------------------------------------------------------------------------------------
def ulp_dtype(ref64, dtype):
    """Spacing of ``dtype`` at |ref| (2^floor(log2 |ref|) * eps); below the smallest normal number, the subnormal
    spacing."""
    fi = torch.finfo(dtype)
    return torch.exp2(torch.floor(torch.log2(ref64.abs().clamp(min=fi.tiny)))) * fi.eps


def check(out, ref64, what, ulps=1.0, floor=None, dtype=None):
    """Every element within ``ulps`` ulps of the fp64 reference plus ``floor``; NaN fails.  Prints the fraction of the
    bound used."""
    dtype = dtype or out.dtype
    err = (out.double() - ref64).abs()
    tol = ulps * ulp_dtype(ref64, dtype) + (0.0 if floor is None else floor)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} outside {ulps} ulp + floor; first at flat index "
                             f"{i}: out {out.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r}")
    used = float((err / tol).max()) if out.numel() else 0.0
    worst = float((err / ulp_dtype(ref64, dtype)).max()) if out.numel() else 0.0
    print(f"[ulp] {what}: max {worst:.3f} ulp, {used:.3f} of the bound")
    return used


def expect_exact(out, ref64, what):
    """``out`` equals the one rounding of the exact result: fp64 -> fp32 (exact by the premise) -> out's dtype."""
    assert out.shape == ref64.shape, (what, tuple(out.shape), tuple(ref64.shape))
    want = ref64.to(FP32).to(out.dtype).double()
    got = out.double()
    bad = torch.isnan(got) | (got != want)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{out.numel()} elements differ from the single rounding of the "
                             f"fp64 result; first at {idx}: out {out[tuple(idx)].item()!r} want "
                             f"{want[tuple(idx)].item()!r} (exact {ref64[tuple(idx)].item()!r})")


def assert_exact_premise(bound, what):
    """``bound`` >= every partial sum's magnitude (sum of |products| + |bias| + |addend|): all of them are exact in fp32."""
    b = float(bound) if not torch.is_tensor(bound) else float(bound.max())
    assert b < EXACT_LIMIT, f"{what}: inputs too large for exact fp32 accumulation ({b:.4g} >= 2^24)"


_SENTINEL = {BF16: 0x7FA5, FP16: 0x7E5A, FP32: 0x7FC05A5A}   # NaN bit patterns no kernel produces
_INT = {2: torch.int16, 4: torch.int32}


def _esz(dtype):
    return torch.finfo(dtype).bits // 8


class Canvas:
    """An output view [rows, cols] inside a buffer of sentinel bits: ``lead`` elements before its base, a pitch gap of
    ``gap`` elements after every row (the pitch stays a multiple of 16 bytes) and ``tail_rows`` rows after the last.
    ``lead`` a multiple of 16 bytes gives an aligned base, one element more a misaligned one."""

    def __init__(self, rows, cols, dtype, *, aligned=True, gap=8, tail_rows=2, init=None, device=DEV):
        unit = 16 // _esz(dtype)
        self.rows, self.cols, self.dtype = rows, cols, dtype
        self.pitch = -(-cols // unit) * unit + gap
        self.lead = 2 * unit + (0 if aligned else 1)
        n = self.lead + (rows + tail_rows) * self.pitch
        self.buf = torch.full((n,), _SENTINEL[dtype], dtype=_INT[_esz(dtype)], device=device).view(dtype)
        self.view = self.buf[self.lead:self.lead + rows * self.pitch].view(rows, self.pitch)[:, :cols]
        if init is not None:
            self.view.copy_(init)

    def check_untouched(self, what, written_rows=None):
        """Every element outside the view (and, with ``written_rows``, every view row from there on) still holds the
        sentinel bits."""
        s = _SENTINEL[self.dtype]
        bits = self.buf.view(_INT[_esz(self.dtype)])
        body = bits[self.lead:].view(-1, self.pitch)
        r = self.rows if written_rows is None else written_rows
        regions = {"bytes before the base": bits[:self.lead], "pitch gap": body[:self.rows, self.cols:],
                   "rows after the view": body[r:]}
        for name, reg in regions.items():
            n = int((reg != s).sum())
            if n:
                raise AssertionError(f"{what}: {n} elements of the {name} were written")


def verify(canvas, ref64, what):
    expect_exact(canvas.view, ref64, what)
    canvas.check_untouched(what)
    print(f"[exact] {what}: {canvas.view.numel()} elements exact, canaries intact")


def poisoned(vals, poison=float("nan")):
    """``vals`` [R, C] copied into a buffer whose pitch gap and two rows before and after hold ``poison``."""
    R, C = vals.shape
    pitch = -(-C // 8) * 8 + 8
    buf = torch.full((R + 4, pitch), poison, dtype=vals.dtype, device=vals.device)
    v = buf[2:2 + R, :C]
    v.copy_(vals)
    return v


def ints(shape, lo, hi, gen, dtype, device=DEV):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=device).to(dtype)


def op_matrix(x, mn):
    """The logical operand [rows, K] of a GEMM input stored K-major ([rows, K]) or MN-major ([K, rows])."""
    return x.t() if mn else x


def mm64(a, b):
    """a [m, K] @ b [n, K]^T in fp64, in K chunks that keep the fp64 copies near 1 GB."""
    K = a.shape[1]
    step = max(64, (1 << 27) // max(a.shape[0], b.shape[0]))
    out = None
    for k0 in range(0, K, step):
        part = a[:, k0:k0 + step].double() @ b[:, k0:k0 + step].double().t()
        out = part if out is None else out + part
    return out


def tile_coords(t, num_m, num_n):
    """The kernels' rasterisation: groups of 8 row tiles, swept column by column."""
    per = GROUP_M * num_n
    g = t // per
    first = g * GROUP_M
    gs = min(GROUP_M, num_m - first)
    r = t - g * per
    return first + r % gs, r // gs


# ---------------------------------------------------------------------------------------------------------------------
# CPU tier: the checkers reject planted faults in an emulation of the kernel
# ---------------------------------------------------------------------------------------------------------------------
FAULTS = ["none", "drop_k16", "swap_halves", "bias_after_cast", "n_tail_shift", "skip_tile", "write_past_n"]


def emulate_dense(a, b, bias, canvas, fault):
    """D = A B^T + bias written tile by tile as the kernel does it (fp32 accumulation over k16 steps, bias in fp32,
    one rounding), with one planted fault."""
    M, K = a.shape
    N = b.shape[0]
    nm, nn = -(-M // TILE_M), -(-N // TILE_N)
    a64, b64, bias32 = a.double(), b.double(), bias.float()
    for t in range(nm * nn):
        tm, tn = tile_coords(t, nm, nn)
        if fault == "skip_tile" and tm == nm - 1 and nm % GROUP_M != 0 and tn == nn - 1:
            continue   # the last tile of the partial raster group
        rows = slice(tm * TILE_M, min(M, tm * TILE_M + TILE_M))
        cols = slice(tn * TILE_N, min(N, tn * TILE_N + TILE_N))
        acc = torch.zeros(rows.stop - rows.start, cols.stop - cols.start, dtype=torch.float64)
        for k0 in range(0, K, 16):
            if fault == "drop_k16" and t == 0 and k0 == 16:
                continue
            acc += a64[rows, k0:k0 + 16] @ b64[cols, k0:k0 + 16].t()
        acc = acc.float()
        if fault == "swap_halves" and t == 0:
            acc = torch.cat([acc[64:128], acc[:64]])
        if fault == "bias_after_cast":
            out = (acc.to(canvas.dtype).float() + bias32[cols]).to(canvas.dtype)
        else:
            out = (acc + bias32[cols]).to(canvas.dtype)
        if fault == "n_tail_shift" and cols.stop == N:
            out[:, -1] = out[:, -2]
        canvas.view[rows, cols] = out
    if fault == "write_past_n":
        canvas.buf[canvas.lead + N] = 0


@pytest.mark.parametrize("fault", FAULTS)
def test_checker_rejects_planted_faults(fault):
    """M = 1100 (a full raster group, then a group of one), N = 520 (a 8-column tail tile), K = 136: the emulated kernel
    passes the exact check and the canaries, every planted fault fails one of them."""
    gen = torch.Generator().manual_seed(0)
    M, N, K = 1100, 520, 136
    a = ints((M, K), -12, 12, gen, BF16, "cpu")
    b = ints((N, K), -12, 12, gen, BF16, "cpu")
    bias = ints((N,), -300, 300, gen, BF16, "cpu")
    ref = a.double() @ b.double().t() + bias.double()
    assert_exact_premise(12 * 12 * K + 300, "emulation")
    canvas = Canvas(M, N, BF16, device="cpu")
    emulate_dense(a, b, bias, canvas, fault)
    if fault == "none":
        verify(canvas, ref, "emulated kernel")
    else:
        with pytest.raises(AssertionError):
            verify(canvas, ref, f"planted fault {fault}")


def test_canvas_layout():
    """The canvas puts aligned views on 16-byte boundaries and misaligned ones one element off, with 16-byte pitches."""
    for dtype in (BF16, FP16, FP32):
        for aligned in (True, False):
            c = Canvas(5, 3, dtype, aligned=aligned, device="cpu")
            assert (c.view.data_ptr() % 16 == 0) == aligned
            assert (c.pitch * _esz(dtype)) % 16 == 0 and c.view.stride(0) == c.pitch
            assert torch.isnan(c.view).all()
            c.check_untouched("fresh canvas")


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers: direct calls of the C ABI (explicit SM count and schedule)
# ---------------------------------------------------------------------------------------------------------------------
def _nat():
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import fp8, moe  # noqa: F401  (register the MX-FP8 and grouped signatures)
    return nat, nat.require()


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def dense(a, b, d, *, a_mn, b_mn, bias=None, c=None, num_sms=None, sched="static"):
    """D = A_op B_op^T (+ bias) (+ C) through ``tb_gemm_bf16_ex``; C may be D (accumulation)."""
    nat, L = _nat()
    M, N = d.shape
    K = a.shape[0] if a_mn else a.shape[1]
    prev = L.tb_gemm_sched_mode(-1)
    L.tb_gemm_sched_mode(1 if sched == "dynamic" else 0)
    try:
        code = L.tb_gemm_bf16_ex(_ptr(a), _ptr(b), d.data_ptr(), _ptr(bias), _ptr(c), M, N, K,
                                 a.stride(0), b.stride(0), d.stride(0),
                                 c.stride(0) if c is not None else 0, int(a_mn), int(b_mn), int(d.dtype == FP32), 1,
                                 num_sms or nat.num_sms(), nat.stream(), int(a.dtype == FP16))
    finally:
        L.tb_gemm_sched_mode(prev)
    nat.check(code, "tb_gemm_bf16_ex")


def swiglu_dense(x, w, h, gu, num_sms=None):
    nat, L = _nat()
    M, K = x.shape
    F = h.shape[1]
    nat.check(L.tb_gemm_swiglu(x.data_ptr(), w.data_ptr(), h.data_ptr(), _ptr(gu), M, F, K, x.stride(0), w.stride(0),
                               h.stride(0), gu.stride(0) if gu is not None else 0, num_sms or nat.num_sms(),
                               nat.stream(), int(x.dtype == FP16)), "tb_gemm_swiglu")


def swiglu_bound(g64, u64, dtype):
    """h = g sigmoid(g) u in fp32 from exact g, u.  fast_sigmoid (ptx.cuh): the rounding of g log2 e costs <= 2^-24 |g|
    log2 e relative in the argument, i.e. <= 2^-24 |g| relative in 2^arg; MUFU ex2 <= 2^-22, 1 + e one rounding, MUFU rcp
    <= 2 ulp, then two fp32 products: <= (|g| + 16) 2^-24 relative in all.  Where sigmoid(g) < 2^-126 the .ftz
    instructions flush it to 0: absolute <= |g u| 2^-126.  Plus 1 ulp of the output."""
    h64 = g64 * torch.sigmoid(g64) * u64
    floor = h64.abs() * (g64.abs() + 16) * 2.0 ** -24 + (g64 * u64).abs() * 2.0 ** -126
    return h64, floor


# ---------------------------------------------------------------------------------------------------------------------
# 1. dense GEMM: exact, covering design (see the module docstring)
# ---------------------------------------------------------------------------------------------------------------------
M_S = [1, 77, 128, 129, 1000, 1100]
N_S = [1, 3, 7, 13, 255, 256, 257, 520]
K_S = [8, 16, 56, 64, 72, 100, 136]
N_STAGED = [256, 520, 136]   # whole 16-byte rows: a full tile, an 8-column tail tile, a partial first tile
EPILOGUES = ["plain", "bias", "addend16", "acc16", "fp32", "fp32_bias", "fp32_acc_view", "fp32_addend"]
INSTANTIATIONS = [(dt, am, bm, path) for dt in ("bf16", "fp16") for am in (0, 1) for bm in (0, 1)
                  for path in ("staged", "register")]


def _dense_case(dtype, a_mn, b_mn, aligned, epi, M, N, K, sched, gen, num_sms=None, lim=12):
    """One exact dense case with canaries; returns nothing, raises on any mismatch."""
    a = poisoned(ints((K, M) if a_mn else (M, K), -lim, lim, gen, dtype))
    b = poisoned(ints((K, N) if b_mn else (N, K), -lim, lim, gen, dtype))
    ref = mm64(op_matrix(a, a_mn), op_matrix(b, b_mn))
    bound = lim * lim * K
    out_dtype = FP32 if epi.startswith("fp32") else dtype
    bias = c = init = None
    if epi in ("bias", "fp32_bias"):
        bias = poisoned(ints((1, N), -300, 300, gen, dtype))[0]   # a read past N meets NaN
        ref, bound = ref + bias.double(), bound + 300
    if epi in ("acc16", "fp32_acc_view"):
        lim_c = 3000 if out_dtype != FP32 else 1 << 20
        init = ints((M, N), -lim_c, lim_c, gen, out_dtype)
        ref, bound = ref + init.double(), bound + lim_c
    canvas = Canvas(M, N, out_dtype, aligned=aligned, init=init, gap=24 if epi == "fp32_acc_view" else 8)
    if init is not None:
        c = canvas.view
    if epi in ("addend16", "fp32_addend"):
        lim_c = 3000 if out_dtype != FP32 else 1 << 20
        c = poisoned(ints((M, N), -lim_c, lim_c, gen, out_dtype))
        ref, bound = ref + c.double(), bound + lim_c
    assert_exact_premise(bound, epi)
    dense(a, b, canvas.view, a_mn=a_mn, b_mn=b_mn, bias=bias, c=c, num_sms=num_sms, sched=sched)
    torch.cuda.synchronize()
    verify(canvas, ref, f"{epi} {dtype} a_mn={a_mn} b_mn={b_mn} {'aligned' if aligned else 'off-by-one'} "
                        f"M={M} N={N} K={K} {sched} sms={num_sms}")


@gpu
@pytest.mark.parametrize("inst", INSTANTIATIONS, ids=lambda p: "-".join(map(str, p)))
def test_dense_exact(inst):
    dt, a_mn, b_mn, path = inst
    j = INSTANTIATIONS.index(inst)
    dtype = BF16 if dt == "bf16" else FP16
    gen = torch.Generator(device=DEV).manual_seed(100 + j)
    for i in range(8):
        _dense_case(dtype, a_mn, b_mn, path == "staged", EPILOGUES[i], M_S[(i + j) % 6], N_S[(i + 3 * j) % 8],
                    K_S[(i + 2 * j) % 7], ("static", "dynamic")[(i + j) % 2], gen)
    if path == "staged":   # the rows of D must end on 16 bytes for the staged epilogue to run
        for i in range(8):
            _dense_case(dtype, a_mn, b_mn, True, EPILOGUES[i], M_S[(i + j + 3) % 6], N_STAGED[(i + j) % 3],
                        K_S[(i + 2 * j + 1) % 7], ("static", "dynamic")[(i + j + 1) % 2], gen)


@gpu
@pytest.mark.parametrize("out", ["fp32", "bf16", "fp32_acc"])
def test_dense_exact_near_2_24(out):
    """Same-signed integers up to 255 over K = 256: sums up to 2^24 - 2^17, which only a full fp32 accumulator keeps;
    fp32 output pins every bit of it, bf16 output the rounding of 24-bit integers."""
    gen = torch.Generator(device=DEV).manual_seed(7)
    M, N, K = 300, 300, 256
    a = poisoned(ints((M, K), 160, 255, gen, BF16) * torch.where(torch.arange(M, device=DEV) % 3 == 0, -1, 1)[:, None]
                 .to(BF16))
    b = poisoned(ints((N, K), 160, 255, gen, BF16))
    assert_exact_premise(255 * 255 * K, "near 2^24")
    ref = mm64(a, b)
    assert float(ref.abs().max()) > 2.0 ** 23
    init = None
    if out == "fp32_acc":
        init = ints((M, N), -(1 << 16), 1 << 16, gen, FP32)
        assert_exact_premise(255 * 255 * K + (1 << 16), "near 2^24 acc")
        ref = ref + init.double()
    canvas = Canvas(M, N, BF16 if out == "bf16" else FP32, init=init)
    dense(a, b, canvas.view, a_mn=0, b_mn=0, c=canvas.view if init is not None else None)
    torch.cuda.synchronize()
    verify(canvas, ref, f"near 2^24 {out}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. the persistent loop: several tiles per CTA, K-block counts that are not multiples of the 4-stage ring
# ---------------------------------------------------------------------------------------------------------------------
PERSIST_K = [40, 128, 136, 320, 384]   # 1, 2, 3, 5, 6 K blocks of 64


@gpu
@pytest.mark.parametrize("epi", ["addend16", "acc16", "fp32_acc_view", "bias", "swiglu"])
def test_persistent_loop_exact(epi):
    """1, 2 or 3 CTAs over 27 tiles (M = 1100, N = 520; SwiGLU: F = 384) under static scheduling: the mbarrier phase
    carried across tiles, the staged buffers reused across tiles and the addend chunks loaded during the next tile's
    mainloop all run many times.  Every case is also run through the register path (D one element off)."""
    gen = torch.Generator(device=DEV).manual_seed(11)
    for i, K in enumerate(PERSIST_K):
        sms = 1 + i % 3
        if epi == "swiglu":
            M, F = 1100, 384
            x = poisoned(ints((M, K), -4, 4, gen, BF16) / 4)   # quarters: |g| stays where sigmoid is not flushed
            w = poisoned(ints((2 * F, K), -3, 3, gen, BF16))
            assert_exact_premise(4 * 3 * K, "swiglu (in units of 1/4)")
            gu64 = mm64(x, w)
            h = Canvas(M, F, BF16)
            gu = Canvas(M, 2 * F, BF16)
            swiglu_dense(x, w, h.view, gu.view, num_sms=sms)
            torch.cuda.synchronize()
            verify(gu, gu64, f"persistent swiglu g|u K={K} sms={sms}")
            h64, floor = swiglu_bound(gu64[:, :F], gu64[:, F:], BF16)
            check(h.view, h64, f"persistent swiglu h K={K} sms={sms}", floor=floor)
            h.check_untouched("persistent swiglu h")
            continue
        for aligned in (True, False):
            _dense_case(BF16 if i % 2 == 0 else FP16, i % 2, (i // 2) % 2, aligned, epi, 1100, 520, K, "static", gen,
                        num_sms=sms)


# ---------------------------------------------------------------------------------------------------------------------
# 3. SwiGLU epilogue (dense, staged): g|u exact, h within its derived bound
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
@pytest.mark.parametrize("write_gu", [False, True])
def test_swiglu_dense_exact(write_gu, dtype):
    gen = torch.Generator(device=DEV).manual_seed(12)
    M, F, K = 1000, 640, 136
    x = poisoned(ints((M, K), -6, 6, gen, dtype) / 4)
    w = poisoned(ints((2 * F, K), -4, 4, gen, dtype))
    assert_exact_premise(6 * 4 * K, "swiglu (in units of 1/4)")
    gu64 = mm64(x, w)
    h = Canvas(M, F, dtype)
    gu = Canvas(M, 2 * F, dtype)
    swiglu_dense(x, w, h.view, gu.view if write_gu else None)
    torch.cuda.synchronize()
    if write_gu:
        verify(gu, gu64, f"swiglu g|u {dtype}")
    else:
        gu.check_untouched("g|u not requested", written_rows=0)
    h64, floor = swiglu_bound(gu64[:, :F], gu64[:, F:], dtype)
    check(h.view, h64, f"swiglu h {dtype} write_gu={write_gu}", floor=floor)
    h.check_untouched("swiglu h")


# ---------------------------------------------------------------------------------------------------------------------
# 4. grouped (mixture-of-experts) GEMMs
# ---------------------------------------------------------------------------------------------------------------------
def group_layout(counts):
    """Padded row offsets and the expert of every 128-row tile of an expert-sorted buffer."""
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + -(-c // TILE_M) * TILE_M)
    tile_expert = [e for e in range(len(counts)) for _ in range((offsets[e + 1] - offsets[e]) // TILE_M)]
    return offsets, tile_expert


def sorted_rows(counts, offsets, cols, lim, gen, dtype, scale=1):
    """[capacity, cols]: expert e's rows at [offsets[e], offsets[e] + counts[e]), zero padding rows, two spare tiles
    (capacity past the device-side tile count) of NaN."""
    cap = offsets[-1] + 2 * TILE_M
    x = torch.full((cap, cols), float("nan"), dtype=dtype, device=DEV)
    x[:offsets[-1]] = 0
    for e, c in enumerate(counts):
        if c:
            x[offsets[e]:offsets[e] + c] = ints((c, cols), -lim, lim, gen, dtype) / scale
    return poisoned(x)


COUNT_PATTERNS = {
    "edges": [0, 1, 127, 128, 129, 255, 0, 300, 2, 0],
    "one_takes_all": [0] * 77 + [1000] + [0] * 50,
    "e128": None,   # 128 experts, random counts with every edge value present
}


def _counts(name, gen):
    if COUNT_PATTERNS[name] is not None:
        return COUNT_PATTERNS[name]
    c = torch.randint(0, 200, (128,), generator=torch.Generator().manual_seed(5)).tolist()
    c[:6] = [0, 1, 127, 128, 129, 0]
    return c


def _index(counts, offsets, tile_expert):
    cap_tiles = offsets[-1] // TILE_M + 2
    te = torch.zeros(cap_tiles, dtype=torch.int32, device=DEV)   # spare tiles name expert 0 (valid, never used)
    if tile_expert:
        te[:len(tile_expert)] = torch.tensor(tile_expert, dtype=torch.int32, device=DEV)
    nmt = torch.tensor([offsets[-1] // TILE_M], dtype=torch.int32, device=DEV)
    off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
    return te, nmt, off


def run_grouped(mode, counts, dtype, gen, N, K, num_sms=None, lim=8):
    """mode: fwd (B [E N, K] K-major), dgrad (B [E K, N] MN-major), swiglu (W_gu [E 2F, K], F = N)."""
    nat, L = _nat()
    E = len(counts)
    offsets, tile_expert = group_layout(counts)
    te, nmt, _ = _index(counts, offsets, tile_expert)
    a = sorted_rows(counts, offsets, K, lim, gen, dtype, scale=4 if mode == "swiglu" else 1)
    cap = a.shape[0]
    sms = num_sms or nat.num_sms()
    f16 = int(dtype == FP16)
    valid = offsets[-1]
    if mode == "swiglu":
        F = N
        w = poisoned(ints((E * 2 * F, K), -3, 3, gen, dtype))
        assert_exact_premise(lim * 3 * K, "grouped swiglu (in units of 1/4)")
        h, gu = Canvas(cap, F, dtype), Canvas(cap, 2 * F, dtype)
        nat.check(L.tb_gemm_grouped_swiglu(a.data_ptr(), w.data_ptr(), h.view.data_ptr(), gu.view.data_ptr(), cap, F, K,
                                           E, a.stride(0), w.stride(0), h.pitch, gu.pitch, te.data_ptr(),
                                           nmt.data_ptr(), sms, nat.stream(), f16), "tb_gemm_grouped_swiglu")
        torch.cuda.synchronize()
        gu64 = torch.zeros(valid, 2 * F, dtype=torch.float64, device=DEV)
        for e in range(E):
            r = slice(offsets[e], offsets[e + 1])
            if r.stop > r.start:
                gu64[r] = mm64(a[r], w[e * 2 * F:(e + 1) * 2 * F])
        expect_exact(gu.view[:valid], gu64, f"grouped swiglu g|u {dtype}")
        gu.check_untouched("grouped swiglu g|u", written_rows=valid)
        h64, floor = swiglu_bound(gu64[:, :F], gu64[:, F:], dtype)
        check(h.view[:valid], h64, f"grouped swiglu h {dtype} E={E}", floor=floor)
        h.check_untouched("grouped swiglu h", written_rows=valid)
        return
    bmn = mode == "dgrad"
    w = poisoned(ints((E * K, N) if bmn else (E * N, K), -lim, lim, gen, dtype))
    assert_exact_premise(lim * lim * K, f"grouped {mode}")
    d = Canvas(cap, N, dtype)
    nat.check(L.tb_gemm_grouped(a.data_ptr(), w.data_ptr(), d.view.data_ptr(), cap, N, K, E, a.stride(0), w.stride(0),
                                d.pitch, int(bmn), te.data_ptr(), nmt.data_ptr(), sms, nat.stream(), f16),
              "tb_gemm_grouped")
    torch.cuda.synchronize()
    ref = torch.zeros(valid, N, dtype=torch.float64, device=DEV)
    for e in range(E):
        r = slice(offsets[e], offsets[e + 1])
        if r.stop > r.start:
            ref[r] = mm64(a[r], w[e * K:(e + 1) * K].t() if bmn else w[e * N:(e + 1) * N])
    expect_exact(d.view[:valid], ref, f"grouped {mode} {dtype} E={E}")
    pad = torch.ones(valid, dtype=torch.bool, device=DEV)
    for e, c in enumerate(counts):
        pad[offsets[e]:offsets[e] + c] = False
    assert bool((d.view[:valid][pad] == 0).all()), "padding rows must be exact zeros"
    d.check_untouched(f"grouped {mode}: rows past the device-side tile count", written_rows=valid)
    print(f"[exact] grouped {mode} {dtype} E={E} sms={sms}: {valid} rows exact, spare tiles untouched")


def run_grouped_wgrad(out, counts, dtype, gen, M, N, num_sms=None, lim=8):
    """D_e [M, N] (+)= dY_e^T X_e over expert e's padded rows; out: fp32, 16 (dY's dtype), fp32_acc, acc16."""
    nat, L = _nat()
    E = len(counts)
    offsets, _ = group_layout(counts)
    _, _, off = _index(counts, offsets, [])
    rows = max(offsets[-1], TILE_M)
    dy = sorted_rows(counts, offsets, M, lim, gen, dtype)[:rows]
    x = sorted_rows(counts, offsets, N, lim, gen, dtype)[:rows]
    out_dtype = FP32 if out.startswith("fp32") else dtype
    acc = out in ("fp32_acc", "acc16")
    lim_c = (1 << 20) if out_dtype == FP32 else 2000
    init = ints((E * M, N), -lim_c, lim_c, gen, out_dtype) if acc else None
    assert_exact_premise(lim * lim * max(max(counts), 1) + (lim_c if acc else 0), "grouped wgrad")
    d = Canvas(E * M, N, out_dtype, init=init, gap=24)
    nat.check(L.tb_gemm_grouped_wgrad(dy.data_ptr(), x.data_ptr(), d.view.data_ptr(), M, N, E, rows, dy.stride(0),
                                      x.stride(0), d.pitch, off.data_ptr(), int(out_dtype == FP32), int(acc),
                                      num_sms or nat.num_sms(), nat.stream(), int(dtype == FP16)),
              "tb_gemm_grouped_wgrad")
    torch.cuda.synchronize()
    ref = init.double() if acc else torch.zeros(E * M, N, dtype=torch.float64, device=DEV)
    for e in range(E):
        r = slice(offsets[e], offsets[e + 1])
        if r.stop > r.start:
            ref[e * M:(e + 1) * M] += mm64(dy[r].t(), x[r].t())
    verify(d, ref, f"grouped wgrad {out} {dtype} E={E} M={M} N={N} sms={num_sms}")


@gpu
@pytest.mark.parametrize("pattern", list(COUNT_PATTERNS))
@pytest.mark.parametrize("mode", ["fwd", "dgrad", "swiglu"])
def test_grouped_exact(mode, pattern):
    """Experts with 0, 1, 127, 128, 129 rows, one expert taking every row, 128 experts; N = 200 and F = 256 (tails of
    the 256 / 128-wide output tiles), K = 136 (a partial K block; dgrad: 192, whole blocks, see DESIGN)."""
    gen = torch.Generator(device=DEV).manual_seed(13)
    counts = _counts(pattern, gen)
    for i, dtype in enumerate((BF16, FP16)):
        if mode == "swiglu":
            run_grouped(mode, counts, dtype, gen, N=256, K=136)
        else:
            run_grouped(mode, counts, dtype, gen, N=200, K=192 if mode == "dgrad" else 136)


@gpu
@pytest.mark.parametrize("pattern", ["edges", "one_takes_all"])
@pytest.mark.parametrize("out", ["fp32", "16", "fp32_acc", "acc16"])
def test_grouped_wgrad_exact(out, pattern):
    """Empty experts are zeroed, or left unchanged when accumulating; M = 200 and N = 136 are tile tails; D is a view
    with a pitch gap."""
    gen = torch.Generator(device=DEV).manual_seed(14)
    for dtype in (BF16, FP16):
        run_grouped_wgrad(out, _counts(pattern, gen), dtype, gen, M=200, N=136)


@gpu
@pytest.mark.parametrize("mode", ["fwd", "dgrad", "swiglu", "wgrad"])
def test_grouped_persistent_loop(mode):
    """1, 2 and 3 CTAs for the whole grouped problem: many tiles (and, for wgrad, many experts' K ranges) per CTA."""
    gen = torch.Generator(device=DEV).manual_seed(15)
    counts = [129, 0, 300, 1, 128, 0, 640, 5]
    for sms in (1, 2, 3):
        if mode == "wgrad":
            run_grouped_wgrad("fp32_acc" if sms != 2 else "16", counts, BF16, gen, M=200, N=300, num_sms=sms)
        elif mode == "swiglu":
            run_grouped(mode, counts, BF16, gen, N=384, K=136, num_sms=sms)
        else:
            run_grouped(mode, counts, BF16, gen, N=520, K=320 if mode == "fwd" else 384, num_sms=sms)


@gpu
def test_grouped_qwen3_moe_shape():
    """Qwen3-30B-A3B: 128 experts, top-8 routing of 2048 tokens, H = 2048, F = 768: gate|up SwiGLU, down (K = 768),
    down dgrad (MN-major B) and down wgrad into fp32."""
    gen = torch.Generator(device=DEV).manual_seed(16)
    E, k, T, H, F = 128, 8, 2048, 2048, 768
    ids = torch.rand(T, E, generator=torch.Generator().manual_seed(3)).topk(k, dim=1).indices
    counts = torch.bincount(ids.reshape(-1), minlength=E).tolist()
    run_grouped("swiglu", counts, BF16, gen, N=F, K=H, lim=4)
    run_grouped("fwd", counts, BF16, gen, N=H, K=F)
    run_grouped("dgrad", counts, BF16, gen, N=F, K=H)
    run_grouped_wgrad("fp32", counts, BF16, gen, M=H, N=F)


# ---------------------------------------------------------------------------------------------------------------------
# 5. MX-FP8
# ---------------------------------------------------------------------------------------------------------------------
def mx_operand(R, K, row_exp, gen):
    """bf16 [R, K] = q 2^(r + u): q an integer in [-8, 8], r one exponent per row in ``row_exp``, u in [0, 3] per
    32-block.  The quantiser represents it exactly (4-bit q times a power of two).  Returns (x, |q| 2^u)."""
    q = torch.randint(-8, 9, (R, K), generator=gen, device=DEV).double()
    r = torch.randint(row_exp[0], row_exp[1] + 1, (R, 1), generator=gen, device=DEV).double()
    u = torch.randint(0, 4, (R, K // 32), generator=gen, device=DEV).double().repeat_interleave(32, 1)
    x = (q * torch.exp2(r + u)).to(BF16)
    assert torch.equal(x.double(), q * torch.exp2(r + u))
    return x, q.abs() * torch.exp2(u), r


MX_CASES = [  # M, N, K, num_sms (None: all), out
    (1100, 200, 640, None, "fp32"),
    (1100, 200, 640, None, "bf16_addend"),
    (129, 1000, 128, 2, "fp32"),
    (300, 257, 384, 3, "bf16_addend"),
    (1, 7, 256, 1, "fp32"),
    (77, 130, 768, 1, "fp32_acc"),
]


@gpu
@pytest.mark.parametrize("case", MX_CASES, ids=lambda c: "-".join(map(str, c)))
def test_mxfp8_exact(case):
    """Per-row exponents over 2^-30 .. 2^30 and per-block exponents 2^0 .. 2^3 (A and B): a wrong scale atom, row or K
    block changes the result by a power of two.  The block sums and their scaled total stay exact (asserted)."""
    from torchacc_b200.ops import fp8
    nat, L = _nat()
    M, N, K, sms, out = case
    gen = torch.Generator(device=DEV).manual_seed(17 + M)
    a, amag, ra = mx_operand(M, K, (-30, 30), gen)
    b, bmag, rb = mx_operand(N, K, (-30, 30), gen)
    aq, _ = fp8.quantize_mxfp8(a)
    bq, _ = fp8.quantize_mxfp8(b)
    assert torch.equal(fp8.dequantize_mxfp8(aq), a.float()) and torch.equal(fp8.dequantize_mxfp8(bq), b.float()), \
        "quantize_mxfp8 is not exact on q 2^s inputs"
    rel = amag @ bmag.t()                       # |partial sums| / 2^(r_a + r_b)
    assert_exact_premise(rel.max() + 2000, "mxfp8")
    ref = fp8.dequantize_mxfp8(aq).double() @ fp8.dequantize_mxfp8(bq).double().t()
    grid = torch.exp2(ra + rb.t())
    out_dtype = BF16 if out.startswith("bf16") else FP32
    c = init = None
    if out == "bf16_addend":
        c = (torch.randint(-2000, 2001, (M, N), generator=gen, device=DEV).double() * grid).to(BF16)
        ref = ref + c.double()
    if out == "fp32_acc":
        init = (torch.randint(-2000, 2001, (M, N), generator=gen, device=DEV).double() * grid).float()
        ref = ref + init.double()
    d = Canvas(M, N, out_dtype, init=init)
    if init is not None:
        c = d.view
    nat.check(L.tb_gemm_mxfp8(aq.q.data_ptr(), aq.sf.data_ptr(), bq.q.data_ptr(), bq.sf.data_ptr(), d.view.data_ptr(),
                              _ptr(c), M, N, K, aq.q.stride(0), bq.q.stride(0), d.pitch,
                              c.stride(0) if c is not None else 0, int(out_dtype == FP32), sms or nat.num_sms(),
                              nat.stream()), "tb_gemm_mxfp8")
    torch.cuda.synchronize()
    verify(d, ref, f"mxfp8 M={M} N={N} K={K} sms={sms} {out}")


# ---------------------------------------------------------------------------------------------------------------------
# 6. the flagship shapes (llama3.2-1b, 8192 tokens; LM head in 4096-token chunks)
# ---------------------------------------------------------------------------------------------------------------------
T_TOK, HID, FFN, VOCAB, QKV = 8192, 2048, 8192, 128256, 64 * (32 + 2 * 8)
SAMPLE_STRIDE = 61   # odd: coprime to 128 and 256, so the sampled rows / columns hit every tile and most residues


def sample_idx(n, tile):
    """Every 61st index plus the first and the last tile in full."""
    last = (n - 1) // tile * tile
    idx = torch.cat([torch.arange(0, n, SAMPLE_STRIDE), torch.arange(0, min(tile, n)), torch.arange(last, n)])
    return torch.unique(idx).to(DEV)


FLAGSHIP = {   # name: (M, N, K, a_mn, b_mn, epilogue)
    "qkv_fwd": (T_TOK, QKV, HID, 0, 0, "plain"),
    "qkv_dgrad": (T_TOK, HID, QKV, 0, 1, "plain"),
    "qkv_wgrad": (QKV, HID, T_TOK, 1, 1, "fp32_acc"),
    "o_proj_residual": (T_TOK, HID, HID, 0, 0, "addend"),
    "down_residual": (T_TOK, HID, FFN, 0, 0, "addend"),
    "lm_logits": (4096, VOCAB, HID, 0, 0, "plain"),
    "lm_dh": (4096, HID, VOCAB, 0, 1, "plain"),
    "lm_dw_two_chunks": (VOCAB, HID, 4096, 1, 1, "fp32_acc2"),
}


def _flagship_operands(name, gen, gaussian):
    M, N, K, a_mn, b_mn, epi = FLAGSHIP[name]
    la, lb = (2, 4) if K > 10000 else (8, 8)
    if gaussian:
        def mk(shape, lim):
            return poisoned(torch.randn(shape, generator=gen, device=DEV).to(BF16))
    else:
        def mk(shape, lim):
            return poisoned(ints(shape, -lim, lim, gen, BF16))
    chunks = 2 if epi == "fp32_acc2" else 1
    ops = [(mk((K, M) if a_mn else (M, K), la), mk((K, N) if b_mn else (N, K), lb)) for _ in range(chunks)]
    return ops, la * lb * K * chunks


def _flagship_run(name, gen, gaussian):
    M, N, K, a_mn, b_mn, epi = FLAGSHIP[name]
    ops, bound = _flagship_operands(name, gen, gaussian)
    out_dtype = FP32 if epi.startswith("fp32") else BF16
    init = c = None
    lim_c = (1 << 20) if out_dtype == FP32 else 1000
    if epi.startswith("fp32_acc"):
        init = (torch.randn(M, N, generator=gen, device=DEV) if gaussian else ints((M, N), -lim_c, lim_c, gen, FP32))
    d = Canvas(M, N, out_dtype, init=init)
    if epi == "addend":
        c = poisoned(torch.randn(M, N, generator=gen, device=DEV).to(BF16) if gaussian
                     else ints((M, N), -lim_c, lim_c, gen, BF16))
    for a, b in ops:
        dense(a, b, d.view, a_mn=a_mn, b_mn=b_mn, c=d.view if init is not None else c)
    torch.cuda.synchronize()
    d.check_untouched(name)

    def ref(rows=None, cols=None, absolute=False):
        r = None
        for a, b in ops:
            A, B = op_matrix(a, a_mn), op_matrix(b, b_mn)
            if rows is not None:
                A = A[rows]
            if cols is not None:
                B = B[cols]
            if absolute:
                A, B = A.abs(), B.abs()
            p = mm64(A, B)
            r = p if r is None else r + p
        extra = init if init is not None else c
        if extra is not None:
            e = extra.double()
            e = e[rows] if rows is not None else e
            e = e[:, cols] if cols is not None else e
            r = r + (e.abs() if absolute else e)
        return r
    return d, ref, bound + (lim_c if (init is not None or c is not None) else 0)


@gpu
@pytest.mark.parametrize("name", list(FLAGSHIP))
def test_flagship_exact(name):
    """Integer operands at the flagship shapes: the sampled rows (every 61st plus the first and last row tile, against
    all columns) and the sampled columns (against all rows) are exact; the canaries hold around the whole output."""
    gen = torch.Generator(device=DEV).manual_seed(18)
    M, N, K, a_mn, b_mn, epi = FLAGSHIP[name]
    d, ref, bound = _flagship_run(name, gen, gaussian=False)
    assert_exact_premise(bound, name)
    rows, cols = sample_idx(M, TILE_M), sample_idx(N, TILE_N)
    expect_exact(d.view[rows], ref(rows=rows), f"{name} sampled rows")
    expect_exact(d.view[:, cols], ref(cols=cols), f"{name} sampled columns")
    print(f"[exact] {name}: {rows.numel()} rows x {N} and {M} x {cols.numel()} columns exact, canaries intact")


@gpu
def test_flagship_gate_up_swiglu_exact():
    """gate|up of the flagship MLP (8192 x 2 * 8192 x 2048) with the SwiGLU epilogue and the g|u output."""
    gen = torch.Generator(device=DEV).manual_seed(19)
    x = poisoned(ints((T_TOK, HID), -2, 2, gen, BF16) / 4)
    w = poisoned(ints((2 * FFN, HID), -2, 2, gen, BF16))
    assert_exact_premise(2 * 2 * HID, "gate|up (in units of 1/4)")
    h, gu = Canvas(T_TOK, FFN, BF16), Canvas(T_TOK, 2 * FFN, BF16)
    swiglu_dense(x, w, h.view, gu.view)
    torch.cuda.synchronize()
    h.check_untouched("gate|up h")
    gu.check_untouched("gate|up g|u")
    rows = sample_idx(T_TOK, TILE_M)
    gu64 = mm64(x[rows], w)
    expect_exact(gu.view[rows], gu64, "gate|up g|u sampled rows")
    h64, floor = swiglu_bound(gu64[:, :FFN], gu64[:, FFN:], BF16)
    check(h.view[rows], h64, "gate|up h sampled rows", floor=floor)
    cols = sample_idx(FFN, TILE_N // 2)
    gcols = mm64(x, w[cols])
    ucols = mm64(x, w[FFN + cols])
    expect_exact(gu.view[:, cols], gcols, "gate|up g sampled columns")
    expect_exact(gu.view[:, FFN + cols], ucols, "gate|up u sampled columns")
    h64, floor = swiglu_bound(gcols, ucols, BF16)
    check(h.view[:, cols], h64, "gate|up h sampled columns", floor=floor)


@gpu
@pytest.mark.parametrize("name", ["qkv_fwd", "qkv_wgrad", "down_residual", "lm_dh"])
def test_flagship_gaussian_precision(name):
    """Gaussian operands.  The kernel adds one m64n256k16 product block per step into fp32 accumulators: K / 16 steps,
    each at most one rounding (2^-24 relative to the running sum if rounded to nearest, 2^-23 if truncated) of a partial
    sum bounded by sum |a b|, one more inside the 16-product step, and at most two for bias and addend: floor
    (K / 16 + 3) 2^-23 (|A| @ |B| + |C|), plus 1 ulp of the output's final rounding."""
    gen = torch.Generator(device=DEV).manual_seed(20)
    M, N, K, a_mn, b_mn, epi = FLAGSHIP[name]
    d, ref, _ = _flagship_run(name, gen, gaussian=True)
    rows = sample_idx(M, TILE_M)
    steps = K // 16 + 3
    check(d.view[rows], ref(rows=rows), f"gaussian {name}", floor=steps * 2.0 ** -23 * ref(rows=rows, absolute=True))


# ---------------------------------------------------------------------------------------------------------------------
# 7. K = 0 and the empty token batch
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("epi", ["plain", "bias", "addend16", "acc16", "fp32", "fp32_bias", "fp32_acc_view"])
def test_dense_k0(epi):
    """An empty reduction: D = bias (+ addend) in fp32 with one rounding, zeros without either, D unchanged when
    accumulating."""
    gen = torch.Generator(device=DEV).manual_seed(21)
    M, N = 77, 257
    out_dtype = FP32 if epi.startswith("fp32") else BF16
    bias = ints((N,), -300, 300, gen, BF16) if "bias" in epi else None
    init = ints((M, N), -3000, 3000, gen, out_dtype) if epi in ("acc16", "fp32_acc_view") else None
    d = Canvas(M, N, out_dtype, init=init, aligned=False)
    c = d.view if init is not None else (poisoned(ints((M, N), -3000, 3000, gen, BF16)) if epi == "addend16" else None)
    ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
    for t in (bias, c):
        if t is not None:
            ref = ref + t.double()
    a = torch.empty(M, 0, dtype=BF16, device=DEV)
    b = torch.empty(N, 0, dtype=BF16, device=DEV)
    dense(a, b, d.view, a_mn=0, b_mn=0, bias=bias, c=c)
    torch.cuda.synchronize()
    verify(d, ref, f"K=0 {epi}")


@gpu
@pytest.mark.parametrize("grad_view", [None, "write", "accumulate"])
def test_linear_zero_tokens(grad_view):
    """linear() on a batch without tokens: forward and backward match F.linear; the weight gradient is zero (written
    into the engine's gradient view, or that view left unchanged when accumulating)."""
    import torch.nn.functional as F
    from torchacc_b200.ops.linear import linear
    torch.manual_seed(22)
    x = torch.randn(2, 0, 64, device=DEV, dtype=BF16, requires_grad=True)
    w = torch.randn(48, 64, device=DEV, dtype=BF16, requires_grad=True)
    bias = torch.randn(48, device=DEV, dtype=BF16, requires_grad=True)
    xr, wr, br = (t.detach().clone().requires_grad_() for t in (x, w, bias))
    gbuf = torch.randn(48, 72, device=DEV)
    before = gbuf.clone()
    if grad_view is not None:
        w._tb_grad_view = gbuf[:, 8:]
        w._tb_grad_ready = grad_view == "accumulate"
    y = linear(x, w, bias)
    yr = F.linear(xr, wr, br)
    assert y.shape == yr.shape == (2, 0, 48)
    y.backward(torch.ones_like(y))
    yr.backward(torch.ones_like(yr))
    assert x.grad.shape == xr.grad.shape and torch.equal(bias.grad, br.grad)
    if grad_view is None:
        assert torch.equal(w.grad, wr.grad)
    else:
        assert w.grad is None
        want = before[:, 8:] if grad_view == "accumulate" else torch.zeros(48, 64, device=DEV)
        assert torch.equal(gbuf[:, 8:], want)
        assert torch.equal(gbuf[:, :8], before[:, :8])
