"""GPU: the main loop of the wgmma GEMM (csrc/gemm.cu) at realistic K, every operand layout, the persistent schedule
and the scatter GEMM, against float64 and against each other bit for bit.

The epilogue contract (tests/test_gemm_epilogue_gpu.py) stops at K = 200; this file covers what a rework of the stage
ring, the scheduler or the store paths can break: K from 8 to 12800 (1 to 200 k-blocks, ring wraps of the 4-stage wide
and the 6-stage narrow tile and their neighbours), MN-major operands (`vllm_gemm_bf16_tn`, the dgrad / wgrad layouts),
one persistent CTA walking every tile, short last rasteriser groups, and `vllm_gemm_bf16_scatter`.

Bound of the fp32 output (no epilogue: bias 0 and scale 1 are exact, so the output is the accumulator):
    |out - ref| <= E = ceil(K / 16) * 2^-23 * (|A| @ |B|^T)          ref, E computed in float64
  - a product of two bf16 values has at most 16 significant bits, so it is exact in fp32: the only error is the fp32
    summation;
  - wgmma adds one k16 step (16 products) to the accumulator at a time and truncates the step's result toward zero: on
    an H100, 99.9 % of the inexact outputs at K = 8 are smaller in magnitude than the exact sum, and positive operands
    lose magnitude at every step.  A truncation loses less than one ulp of the step's result, at most 2^-23 of the
    magnitude sum sum_k |a b|, so E allows each of the ceil(K / 16) steps 2^-23 * sum_k |a b|.  (The epilogue
    contract's accumulator term has 2^-24, half an ulp per step: the one-step errors measured at K = 8 and 16 on normal
    operands reach 0.91 of this E, 1.83 of that one.)
  - no max|ref| term: a lost or duplicated k-block, a stale stage or a pitch gap read as data moves an element by a
    whole k-block's contribution, orders of magnitude above E.
The bf16 output must equal the fp32 output of the same call rounded to bf16 (RN), bit for bit: both run the same
epilogue on the same accumulator.  It must also round the float64 reference within E (`bf16_rounding.rounds`: RN_bf16
of the reference wherever no rounding midpoint lies within E of it).

Exact integer probe: operands are integers in [-8, 8], so every product has magnitude <= 64 and every partial sum, in
any order and under any truncation, is an integer of magnitude <= 64 K < 2^24 -- exact in fp32.  The fp32 output must
then equal the float64 product exactly and the bf16 output must be its correctly rounded value: a dropped, duplicated or
stale k-block cannot hide inside a tolerance.

Every operand carries NaN wherever the kernel must not read: the pitch gap of a K-major operand (columns K..ld), the
pitch gap of an MN-major one (columns M|N..ld) and 64 rows past K.  Every output is a NaN-prefilled view, with a row
pitch above N and one more row, of a buffer filled with a sentinel: every element of C must be finite and every byte
outside it unchanged.

`pytest -rP -s` prints the worst err / E per entry point, tile width and output type.  On an NVIDIA H100 80GB HBM3 at
700 W it is 0.92 for the fp32 output and 0.04 for the bf16 output, the same for every entry point and tile width (their
outputs are bit-identical, test 2).

The scatter GEMM runs the bf16 epilogue with bias 0 and scale 1 on the same accumulator as a plain `ops.linear` under
the 128 x 256 tile, so every slot must equal the matching rows of `ops.linear` bit for bit; through that identity the
fp64 bound above carries over.  Its flags are read back after a device synchronise and compared on the host: no test
here waits on a count produced by the code under test.
"""
import ctypes
import functools
import math
from types import SimpleNamespace

import pytest
import torch

from visionllm_b200 import _lib
from bf16_rounding import REPORT, U, print_report, rn_bf16, rounds, within

gpu = pytest.mark.gpu
EINVAL, EUNSUPPORTED, EALIGN = -1, -2, -3
NAN = float("nan")
SENTINEL = 4320.0                                   # exact in bf16 and fp32; no output of these tests equals it
FLAG_SENTINEL = 0x5A5A5A5A
TILES = {"1": _lib.GEMM_NARROW_TILE, "2": _lib.GEMM_WIDE_TILE}     # tile width in 128-column units
# entry points: (TA, TB) of vllm_gemm_bf16_tn, or vllm_gemm_bf16 through ops.linear (K-major operands)
LAYOUTS = {"linear": (0, 0), "tn00": (0, 0), "tn01": (0, 1), "tn10": (1, 0), "tn11": (1, 1)}
INT_MAX = 8                                         # integer probe operands lie in [-INT_MAX, INT_MAX]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("GEMM main loop")


# ---------------------------------------------------------------------------------------------------------------------
# helpers (device-agnostic; their CPU cases follow)
# ---------------------------------------------------------------------------------------------------------------------
def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int32: torch.int32}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def integer_sums_exact(K, vmax=INT_MAX):
    """Integer operands in [-vmax, vmax]: is every partial sum of K products exact in fp32, in any order and under any
    truncation?  Each is an integer of magnitude <= vmax^2 K; fp32 holds every integer below 2^24."""
    return vmax * vmax * K < 2 ** 24


def acc_bound(a, b):
    """E of the module docstring for a [M, K] . b [N, K]^T (float64): one truncation per k16 step."""
    return math.ceil(a.shape[1] / 16) * 2 * U * (a.double().abs() @ b.double().abs().T)


def _pitch(cols, dtype, extra=1):
    """A row pitch of at least cols + extra elements, 16-byte aligned."""
    per16 = 16 // torch.tensor([], dtype=dtype).element_size()
    return (cols + extra + per16 - 1) // per16 * per16


def k_major(t, gap=24):
    """t [rows, K] stored K-major: a [rows + 1, ld >= K + gap] buffer of NaN holding t; returns the [rows, K] view."""
    rows, K = t.shape
    buf = torch.full((rows + 1, _pitch(K, t.dtype, gap)), NAN, dtype=t.dtype, device=t.device)
    buf[:rows, :K] = t
    return buf[:rows, :K]


def mn_major(t):
    """t [rows, K] stored MN-major: a [K + 64, ld > rows] buffer of NaN holding t^T; returns the [K, rows] view.  A box
    that reads past row K or column `rows` into the buffer meets NaN."""
    rows, K = t.shape
    buf = torch.full((K + 64, _pitch(rows, t.dtype, 8)), NAN, dtype=t.dtype, device=t.device)
    buf[:K, :rows] = t.T
    return buf[:K, :rows]


class Guarded:
    """A [rows, cols] view with row pitch ld > cols (16-byte aligned) at the top left of a [rows + 1, ld] buffer filled
    with `fill`; the view itself is prefilled with NaN.  `check()`: every element of the view is finite (written) and
    every byte outside it is unchanged."""

    def __init__(self, rows, cols, dtype, device="cuda", fill=SENTINEL):
        self.buf = torch.full((rows + 1, _pitch(cols, dtype)), fill, dtype=dtype, device=device)
        self.view = self.buf[:rows, :cols]
        self.view.fill_(NAN)
        self.outside = torch.ones(self.buf.shape, dtype=torch.bool, device=device)
        self.outside[:rows, :cols] = False
        self.before = bits(self.buf).clone()

    def check(self, what):
        fin = self.view.isfinite()
        assert bool(fin.all()), f"{what}: {int((~fin).sum())} / {fin.numel()} elements of C unwritten or not finite"
        changed = (bits(self.buf) != self.before) & self.outside
        assert not bool(changed.any()), \
            f"{what}: {int(changed.sum())} elements outside C changed, first at {tuple(changed.nonzero()[0].tolist())}"


class Slots:
    """Scatter destinations: n_dst [R, N] slots with row pitch ldc inside one bf16 buffer of sentinels, GAP sentinel rows
    before, between and after them; the slots are NaN-prefilled.  Flags: one int32 word per destination, 256 bytes
    apart, starting at 0, in the middle of a page of sentinel words."""
    GAP = 2
    FLAG_STRIDE, FLAG_OFF = 64, 32                  # words: 256 bytes apart, 128 bytes into each 256-byte block

    def __init__(self, n_dst, R, N, ldc, device="cuda"):
        self.n_dst, self.R, self.N = n_dst, R, N
        G = self.GAP
        self.buf = torch.full((G + n_dst * (R + G), ldc), SENTINEL, dtype=torch.bfloat16, device=device)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=device)
        self.slots = []
        for d in range(n_dst):
            r0 = G + d * (R + G)
            self.slots.append(self.buf[r0:r0 + R, :N])
            self.inside[r0:r0 + R, :N] = True
        self.page = torch.full((1024,), FLAG_SENTINEL, dtype=torch.int32, device=device)
        self.flag_idx = [self.FLAG_STRIDE * d + self.FLAG_OFF for d in range(n_dst)]
        self.page[self.flag_idx] = 0
        self.page_before = self.page.clone()
        self.refill()
        self.before = bits(self.buf).clone()

    def refill(self):
        for s in self.slots:
            s.fill_(NAN)

    def dst(self, d):
        return self.slots[d].data_ptr()

    def flag(self, d):
        return self.page.data_ptr() + 4 * self.flag_idx[d]

    def check(self, ref, passes, tiles_per_pass, what):
        """Slot d == ref rows [d R, (d + 1) R) bit for bit (ref=None: slots untouched); nothing outside the slots
        changed; flag d == passes * tiles_per_pass; every other word of the flag page unchanged."""
        for d, s in enumerate(self.slots):
            if ref is None:
                assert bool(s.isnan().all()), f"{what}: slot {d} was written"
            else:
                want = ref[d * self.R:(d + 1) * self.R]
                diff = bits(s) != bits(want)
                assert not bool(diff.any()), \
                    f"{what}: slot {d}: {int(diff.sum())} / {diff.numel()} elements differ from ops.linear, " \
                    f"first at {tuple(diff.nonzero()[0].tolist())}"
        changed = (bits(self.buf) != self.before) & ~self.inside
        assert not bool(changed.any()), \
            f"{what}: {int(changed.sum())} elements outside the slots changed, first at {tuple(changed.nonzero()[0].tolist())}"
        flags = self.page[self.flag_idx].tolist()
        assert flags == [passes * tiles_per_pass] * self.n_dst, \
            f"{what}: flags {flags}, want {passes} x {tiles_per_pass} each"
        others = torch.ones(self.page.shape, dtype=torch.bool, device=self.page.device)
        others[self.flag_idx] = False
        assert torch.equal(self.page[others], self.page_before[others]), f"{what}: a word of the flag page beside the flags changed"


def scatter_tiles_per_pass(R, N):
    """Flag arrivals per destination and pass: one per consumer warp (8) per 128 x 256 tile of its R rows."""
    return (R // 128) * ((N + 255) // 256) * 8


# ---------------------------------------------------------------------------------------------------------------------
# CPU cases of the helpers
# ---------------------------------------------------------------------------------------------------------------------
def test_integer_probe_precondition():
    assert integer_sums_exact(12800) and integer_sums_exact(2 ** 18 - 1)
    assert not integer_sums_exact(2 ** 18)                          # 64 K = 2^24: the first integer fp32 may not hold
    g = torch.Generator().manual_seed(0)
    K = 12800
    a = torch.randint(-INT_MAX, INT_MAX + 1, (3, K), generator=g).to(torch.bfloat16)
    b = torch.randint(-INT_MAX, INT_MAX + 1, (4, K), generator=g).to(torch.bfloat16)
    a[0] = INT_MAX                                                  # the extreme row: every product +64
    b[0] = INT_MAX
    ref = a.double() @ b.double().T
    assert ref[0, 0] == 64 * K
    # fp32 sums in two different orders (one k16 step at a time, and backwards) are exact
    prod = a.float()[:, None, :] * b.float()[None, :, :]
    steps = prod.view(3, 4, K // 16, 16).sum(-1)
    fwd = torch.zeros(3, 4)
    for j in range(K // 16):
        fwd += steps[..., j]
    bwd = prod.flip(-1).cumsum(-1, dtype=torch.float32)[..., -1]
    assert torch.equal(fwd.double(), ref) and torch.equal(bwd.double(), ref)


def test_bound_on_hand_built_inputs():
    a = torch.tensor([[1.0, -2.0, 0.5, 4.0]], dtype=torch.bfloat16)
    b = torch.tensor([[3.0, 1.0, -8.0, 0.25], [0.0, 0.0, 0.0, 0.0]], dtype=torch.bfloat16)
    E = acc_bound(a, b)
    assert E.dtype == torch.float64
    assert torch.equal(E, torch.tensor([[(3 + 2 + 4 + 1) * 2.0 ** -23, 0.0]], dtype=torch.float64))   # one k16 step
    a17 = torch.full((1, 17), -0.5, dtype=torch.bfloat16)
    b17 = torch.full((1, 17), 3.0, dtype=torch.bfloat16)
    assert acc_bound(a17, b17).item() == 2 * 17 * 1.5 * 2.0 ** -23                              # two k16 steps
    # the integer probe with one k-block dropped or duplicated is far outside E; a full ulp per step is inside
    K = 640
    a = torch.randint(-INT_MAX, INT_MAX + 1, (5, K), generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    b = torch.randint(-INT_MAX, INT_MAX + 1, (6, K), generator=torch.Generator().manual_seed(2)).to(torch.bfloat16)
    ref = a.double() @ b.double().T
    E = acc_bound(a, b)
    within(ref - E, ref, E, "cpu")
    kb = a.double()[:, 128:192] @ b.double()[:, 128:192].T
    for wrong in (ref - kb, ref + kb):
        assert (kb.abs() > E).any()
        with pytest.raises(AssertionError):
            within(wrong, ref, E, "cpu")
    REPORT.pop("cpu", None)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_guard_catches_a_single_changed_byte(dtype):
    o = Guarded(5, 13, dtype, device="cpu")
    assert o.buf.shape[1] > 13 and o.buf.shape[1] * o.buf.element_size() % 16 == 0
    with pytest.raises(AssertionError, match="unwritten"):
        o.check("nothing written")
    o.view.fill_(1.0)
    o.check("every element written")
    o.view[4, 12] = NAN
    with pytest.raises(AssertionError, match="unwritten"):
        o.check("one element unwritten")
    o.view[4, 12] = 2.0
    raw = o.buf.view(torch.uint8)
    esz = o.buf.element_size()
    for r, c in ((0, 13), (4, o.buf.shape[1] - 1), (5, 0)):          # pitch gap of the first / last row, the extra row
        raw[r, c * esz] ^= 1
        with pytest.raises(AssertionError, match="outside C"):
            o.check(f"byte of ({r}, {c})")
        raw[r, c * esz] ^= 1
    o.check("restored")


def test_slot_checker_catches_a_single_changed_byte():
    R, N, ldc = 128, 64, 128
    s = Slots(2, R, N, ldc, device="cpu")
    ref = torch.randn(2 * R, N).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="differ"):
        s.check(ref, 0, 8, "nothing written")
    s.check(None, 0, 8, "untouched")
    for d in range(2):
        s.slots[d].copy_(ref[d * R:(d + 1) * R])
    s.page[s.flag_idx] = 8
    s.check(ref, 1, 8, "one pass")
    raw = s.buf.view(torch.uint8)
    for r, c in ((0, 0), (Slots.GAP, 2 * N), (Slots.GAP + R, 7), (raw.shape[0] - 1, 2 * ldc - 1)):
        raw[r, c] ^= 0x10                           # a gap row, the pitch of a slot row, between slots, the last byte
        with pytest.raises(AssertionError, match="outside the slots"):
            s.check(ref, 1, 8, f"byte ({r}, {c})")
        raw[r, c] ^= 0x10
    raw[Slots.GAP + R + Slots.GAP, 0] ^= 1          # a byte inside slot 1
    with pytest.raises(AssertionError, match="slot 1"):
        s.check(ref, 1, 8, "slot byte")
    raw[Slots.GAP + R + Slots.GAP, 0] ^= 1
    pb = s.page.view(torch.uint8)
    pb[4 * (s.flag_idx[1] + 1)] ^= 1                # the byte after flag 1
    with pytest.raises(AssertionError, match="flag page"):
        s.check(ref, 1, 8, "page byte")
    pb[4 * (s.flag_idx[1] + 1)] ^= 1
    s.page[s.flag_idx[0]] = 7
    with pytest.raises(AssertionError, match="flags"):
        s.check(ref, 1, 8, "short count")


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def stream():
    return torch.cuda.current_stream().cuda_stream


def ops():
    from visionllm_b200 import ops as o
    return o


def gemm_tn(a, a_mn, b, b_mn, out):
    """vllm_gemm_bf16_tn into `out` (a pitched view): a is [M, K] or, MN-major, [K, M]; b is [N, K] or [K, N]."""
    M, N = out.shape
    K = a.shape[0] if a_mn else a.shape[1]
    return _lib.lib().vllm_gemm_bf16_tn(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
                                        out.data_ptr(), out.stride(0), M, N, K, int(out.dtype == torch.float32), stream())


@functools.lru_cache(maxsize=None)
def problem(M, N, K, integer):
    """A [M, K], B [N, K] bf16 (integers in [-8, 8] or normal), each stored K-major and MN-major with NaN around it."""
    g = torch.Generator(device="cuda").manual_seed(M * 1000003 + N * 1009 + K * 2 + int(integer))
    if integer:
        assert integer_sums_exact(K)
        A = torch.randint(-INT_MAX, INT_MAX + 1, (M, K), device="cuda", generator=g).bfloat16()
        B = torch.randint(-INT_MAX, INT_MAX + 1, (N, K), device="cuda", generator=g).bfloat16()
    else:
        A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        B = torch.randn(N, K, device="cuda", generator=g).bfloat16()
    return SimpleNamespace(M=M, N=N, K=K, a={0: k_major(A), 1: mn_major(A)}, b={0: k_major(B), 1: mn_major(B)},
                           ref=A.double() @ B.double().T, E=None if integer else acc_bound(A, B))


def run(layout, p, tile, dtype):
    """C = A . B^T of problem p through one entry point and tile width into a guarded output; returns the view."""
    what = f"{layout} tile {tile} {dtype} M={p.M} N={p.N} K={p.K}"
    out = Guarded(p.M, p.N, dtype)
    ta, tb = LAYOUTS[layout]
    with _lib.knob("gemm_set_variant", TILES[tile]):
        if layout == "linear":
            ops().linear(p.a[0], p.b[0], out=out.view)
        else:
            rc = gemm_tn(p.a[ta], ta, p.b[tb], tb, out.view)
            assert rc == 0, f"{what}: rc {rc}"
    out.check(what)
    return out.view, what


# ---------------------------------------------------------------------------------------------------------------------
# 1. the main loop against fp64, every operand layout
# ---------------------------------------------------------------------------------------------------------------------
# K below one k-block, at and around one; k-block counts at and around the ring sizes (4 stages wide, 6 narrow: 3..7,
# 12 / 13, 24 / 25), each whole and with a ragged last k-block; the product's long K (ViT 3200, wgrad 8192 tokens,
# fc2 12800) and 12800 with a ragged last k-block
KB_COUNTS = (3, 4, 5, 6, 7, 12, 13, 24, 25)
MAIN_K = [8, 16, 56, 64, 72] + sorted({64 * n for n in KB_COUNTS} | {64 * n - 40 for n in KB_COUNTS}) + \
         [3200, 8192, 12792, 12800]
SWEEP_MN = (200, 257)                              # two row-blocks, N one past a multiple of 128 and 256
# one row, N = 8 / 13 (one 16-byte run, an odd tail), ragged M, and 10 row-blocks x 3 wide / 5 narrow column-blocks
SHAPES = [(1, 8), (1, 13), (77, 200), (300, 257), (1153, 520)]
SHAPE_K = (72, 1000)


def main_cases():
    return [(*SWEEP_MN, K) for K in MAIN_K] + [(M, N, K) for (M, N) in SHAPES for K in SHAPE_K]


@gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_main_loop_vs_fp64(layout):
    """fp32 output within E of the fp64 product, bf16 output == the fp32 output rounded and within E of the product
    after one rounding; every K of MAIN_K and every shape, both tile widths."""
    for M, N, K in main_cases():
        p = problem(M, N, K, False)
        for tile in TILES:
            o32, what = run(layout, p, tile, torch.float32)
            o16, _ = run(layout, p, tile, torch.bfloat16)
            within(o32, p.ref, p.E, f"{layout} tile {tile} fp32", what)
            assert same_bits(o16, o32.to(torch.bfloat16)), \
                f"{what}: bf16 output != fp32 output rounded ({int((bits(o16) != bits(o32.bfloat16())).sum())} elements)"
            rounds(o16, p.ref, p.E, f"{layout} tile {tile} bf16", what)


@gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_integer_probe_is_exact(layout):
    """Integer operands in [-8, 8]: fp32 output == the fp64 product exactly, bf16 output == RN_bf16 of it, at every K
    of MAIN_K and every shape, both tile widths."""
    for M, N, K in main_cases():
        p = problem(M, N, K, True)
        for tile in TILES:
            o32, what = run(layout, p, tile, torch.float32)
            o16, _ = run(layout, p, tile, torch.bfloat16)
            bad = o32.double() != p.ref
            assert not bool(bad.any()), (
                f"{what}: {int(bad.sum())} / {bad.numel()} integer sums inexact, first at "
                f"{tuple(bad.nonzero()[0].tolist())}: {o32[bad][0].item()} vs {p.ref[bad][0].item()}")
            assert torch.equal(o16.double(), rn_bf16(p.ref)), f"{what}: bf16 output is not RN_bf16 of the exact sum"


# ---------------------------------------------------------------------------------------------------------------------
# 2. bit-identities between layouts, tile widths and entry points
# ---------------------------------------------------------------------------------------------------------------------
IDENTITY_CASES = [(*SWEEP_MN, K) for K in (8, 72, 64 * 13 - 40, 64 * 24, 3200, 12792)] + [(1, 13, 1000), (1153, 520, 1000)]


@gpu
@pytest.mark.parametrize("M,N,K", IDENTITY_CASES)
def test_layouts_tiles_and_entry_points_are_bit_identical(M, N, K):
    """An MN-major operand gives the bytes of the K-major call on the transposed copy (same MMAs, same k order; only
    the descriptors and tensor maps differ); the 256-column tile gives the bytes of the 128-column one for every
    layout; gemm_tn(0, 0) gives the bytes of ops.linear.  fp32 and bf16 output."""
    p = problem(M, N, K, False)
    for dtype in (torch.float32, torch.bfloat16):
        out = {(lay, t): run(lay, p, t, dtype)[0] for lay in LAYOUTS for t in TILES}
        for lay in LAYOUTS:
            assert same_bits(out[lay, "2"], out[lay, "1"]), f"{lay} {dtype}: 256- and 128-column tiles differ"
        for t in TILES:
            for lay in ("tn01", "tn10", "tn11"):
                assert same_bits(out[lay, t], out["tn00", t]), f"{lay} tile {t} {dtype}: MN-major differs from K-major"
            assert same_bits(out["tn00", t], out["linear", t]), f"tile {t} {dtype}: gemm_tn(0, 0) differs from ops.linear"


# ---------------------------------------------------------------------------------------------------------------------
# 3. the persistent schedule
# ---------------------------------------------------------------------------------------------------------------------
SCHED_M = (1100, 2100)                               # 9 and 17 row-blocks: rasteriser groups of 8 with a last group of 1
SCHED_K = (64, 3 * 64 - 24, 5 * 64, 7 * 64 - 24, 13 * 64)      # 1, 3, 5, 7, 13 k-blocks
SCHED_N = 520


@functools.lru_cache(maxsize=None)
def sched_problem(M, K):
    g = torch.Generator(device="cuda").manual_seed(M + 7 * K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    B = (torch.randn(SCHED_N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(SCHED_N, device="cuda", generator=g).bfloat16()
    res = torch.randn(M, SCHED_N, device="cuda", generator=g).bfloat16()
    return dict(a={0: k_major(A), 1: mn_major(A)}, b={0: k_major(B), 1: mn_major(B)}, bias=bias, res=res)


@gpu
@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("kind", ["tn00", "tn11", "linear_bias_gelu_residual"])
def test_sm_budget_is_bit_identical(kind, tile):
    """One CTA walking every tile (and 2 / 7 CTAs) carries the stage ring's stage and phase across tiles of 1 to 13
    k-blocks: the bytes of the default launch, for 9 and 17 row-blocks (short last rasteriser groups)."""
    def call(p, M, K, dtype, what):
        out = Guarded(M, SCHED_N, dtype)
        if kind == "linear_bias_gelu_residual":
            ops().linear(p["a"][0], p["b"][0], bias=p["bias"], act="gelu", residual=p["res"], out=out.view)
        else:
            t = int(kind == "tn11")
            assert gemm_tn(p["a"][t], t, p["b"][t], t, out.view) == 0
        out.check(what)
        return out.view

    with _lib.knob("gemm_set_variant", TILES[tile]):
        for M in SCHED_M:
            for K in SCHED_K:
                p = sched_problem(M, K)
                for dtype in (torch.float32, torch.bfloat16):
                    what = f"{kind} tile {tile} {dtype} M={M} K={K}"
                    full = call(p, M, K, dtype, what)
                    for n in (1, 2, 7):
                        with _lib.knob("gemm_set_sm_limit", n, 0):
                            got = call(p, M, K, dtype, f"{what} SM budget {n}")
                        diff = bits(got) != bits(full)
                        assert not bool(diff.any()), (f"{what}: SM budget {n} differs from the default grid in "
                                                      f"{int(diff.sum())} elements, first at {tuple(diff.nonzero()[0].tolist())}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the scatter GEMM
# ---------------------------------------------------------------------------------------------------------------------
def scatter(A, B, slots, n_dst=None, R=None, ldc=None, N=None, K=None, lda=None, dst=None, flags=None):
    n_dst = slots.n_dst if n_dst is None else n_dst
    dst = [slots.dst(d) for d in range(slots.n_dst)] if dst is None else dst
    flags = [slots.flag(d) for d in range(slots.n_dst)] if flags is None else flags
    arr = lambda ps: (ctypes.c_void_p * max(len(ps), 1))(*[ctypes.c_void_p(p) for p in ps])   # noqa: E731
    return _lib.lib().vllm_gemm_bf16_scatter(
        A.data_ptr(), A.stride(0) if lda is None else lda, B.data_ptr(), B.stride(0), arr(dst), arr(flags), n_dst,
        slots.R if R is None else R, slots.buf.stride(0) if ldc is None else ldc, slots.N if N is None else N,
        A.shape[1] if K is None else K, stream())


# (n_dst, rows per destination, N, K, ldc - N): every value of each axis at least once, N % 256 != 0 (partial last
# tile) with both pitches
SCATTER_CASES = [(1, 128, 64, 64, 0), (1, 384, 4160, 72, 64), (2, 128, 320, 1024, 64), (2, 384, 4096, 4096, 0),
                 (3, 128, 4160, 4096, 64), (3, 384, 64, 72, 64), (8, 128, 320, 72, 0), (8, 384, 4096, 1024, 64),
                 (8, 128, 4160, 64, 0), (2, 384, 320, 4096, 64)]


@gpu
@pytest.mark.parametrize("n_dst,R,N,K,ldc_extra", SCATTER_CASES)
def test_scatter_slots_and_flags(n_dst, R, N, K, ldc_extra):
    """Slot d == rows [d R, (d + 1) R) of ops.linear under the wide tile, bit for bit, after each of three passes, under
    the narrow tile and under scatter SM budgets of 1 and 3; nothing outside the slots (gap rows, columns N..ldc) or
    beside the flags changes; flag d counts 8 arrivals per 128 x 256 tile per pass."""
    M = n_dst * R
    g = torch.Generator(device="cuda").manual_seed(n_dst * 100 + R + N + K)
    A = k_major(torch.randn(M, K, device="cuda", generator=g).bfloat16())       # NaN pitch gap and row after A
    B = k_major((torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16())
    with _lib.knob("gemm_set_variant", _lib.GEMM_WIDE_TILE):
        ref = ops().linear(A, B)
    assert bool(ref.isfinite().all())
    s = Slots(n_dst, R, N, N + ldc_extra)
    tpp = scatter_tiles_per_pass(R, N)
    passes = 0
    runs = [("pass 1", None), ("pass 2", None), ("pass 3", None),
            ("narrow tile", ("gemm_set_variant", _lib.GEMM_NARROW_TILE)),
            ("scatter SM budget 1", ("gemm_set_sm_limit", 0, 1)),
            ("scatter SM budget 3", ("gemm_set_sm_limit", 0, 3))]
    for what, knob in runs:
        s.refill()
        if knob is None:
            rc = scatter(A, B, s)
        else:
            with _lib.knob(*knob):
                rc = scatter(A, B, s)
        assert rc == 0, f"{what}: rc {rc}"
        passes += 1
        torch.cuda.synchronize()
        s.check(ref, passes, tpp, f"n_dst={n_dst} R={R} N={N} K={K} ldc=N+{ldc_extra} {what}")


@gpu
def test_scatter_rejections_leave_slots_and_flags_untouched():
    """Every documented rejection returns its code before any launch: the slots stay NaN, the flags 0."""
    n_dst, R, N, K = 2, 128, 320, 72
    g = torch.Generator(device="cuda").manual_seed(5)
    A = k_major(torch.randn(n_dst * R, K, device="cuda", generator=g).bfloat16())
    B = k_major(torch.randn(N, K, device="cuda", generator=g).bfloat16())
    s = Slots(n_dst, R, N, N + 64)
    dst = [s.dst(d) for d in range(n_dst)]
    flags = [s.flag(d) for d in range(n_dst)]
    cases = [
        ("n_dst 0", EINVAL, dict(n_dst=0)),
        ("n_dst 9", EINVAL, dict(n_dst=9, dst=dst * 5, flags=flags * 5)),
        ("rows_per_dst % 128", EUNSUPPORTED, dict(R=64)),
        ("N % 64", EUNSUPPORTED, dict(N=96)),
        ("K 0", EINVAL, dict(K=0)),
        ("K < 0", EINVAL, dict(K=-64)),
        ("lda < K", EINVAL, dict(lda=K - 8)),
        ("ldc < N", EINVAL, dict(ldc=N - 8)),
        ("ldc % 8", EALIGN, dict(ldc=N + 4)),
        ("misaligned dst[1]", EALIGN, dict(dst=[dst[0], dst[1] + 2])),
        ("null dst[0]", EINVAL, dict(dst=[0, dst[1]])),
        ("null dst[1]", EINVAL, dict(dst=[dst[0], 0])),
        ("null flags[1]", EINVAL, dict(flags=[flags[0], 0])),
    ]
    for what, code, kw in cases:
        rc = scatter(A, B, s, **kw)
        torch.cuda.synchronize()
        assert rc == code, f"{what}: rc {rc}, want {code}"
        s.check(None, 0, 0, what)


@gpu
def test_scatter_through_peer_comm_counts_recv_flag():
    """PeerComm.virtual: after one and two o_proj passes of every rank, each rank's _RECV_FLAG counter holds exactly
    passes * W * tiles_per_pass (the count the reduce kernel waits for) and receive slot s holds rank s's rows of
    ops.linear bit for bit.  The counters are read back, never waited on."""
    from visionllm_b200 import tp
    W, R, H, K = 3, 384, 4160, 1024
    comms = tp.PeerComm.virtual(W, W * R, H)
    assert all(c.tiles_per_pass == scatter_tiles_per_pass(R, H) for c in comms)
    g = torch.Generator(device="cuda").manual_seed(9)
    ctxs = [torch.randn(W * R, K, device="cuda", generator=g).bfloat16() for _ in range(W)]
    ws = [(torch.randn(H, K, device="cuda", generator=g) / K ** 0.5).bfloat16() for _ in range(W)]
    with _lib.knob("gemm_set_variant", _lib.GEMM_WIDE_TILE):
        refs = [ops().linear(a, w) for a, w in zip(ctxs, ws)]
    for passes in (1, 2):
        for c in comms:
            c.recv.fill_(NAN)
        for c, a, w in zip(comms, ctxs, ws):
            c.oproj_scatter(a, w)
        torch.cuda.synchronize()
        for d, c in enumerate(comms):
            raw = torch.as_tensor(tp._DeviceBytes(c._own, 4096), device="cuda").view(torch.int32)
            flag = int(raw[tp._RECV_FLAG // 4].item())
            assert flag == passes * W * c.tiles_per_pass, f"rank {d} pass {passes}: _RECV_FLAG {flag}"
            for s_ in range(W):
                assert same_bits(c.recv[s_], refs[s_][d * R:(d + 1) * R]), f"rank {d} slot {s_} pass {passes}"
