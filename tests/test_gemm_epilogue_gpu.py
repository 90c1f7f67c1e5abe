"""GPU: every epilogue path of the wgmma GEMM (csrc/gemm.cu) against a float64 reference of the same op on the same
bf16 inputs, and the bit-identities that tie its store paths, schedules and entry points together.

The epilogue has two store paths.  Whole 64-column bf16 chunks are staged in shared memory and leave as 128-byte row
runs; fp32 output, SwiGLU and the last chunk of a ragged N store pairs straight from the accumulator fragments (one
element when N is odd).  Both run the same epilogue arithmetic on the same fp32 accumulator, so the tight fp32 check
below carries over to the staged path through `bf16 output == fp32 output rounded to bf16`, bit for bit.

Bound of the fp32 output (y = acc + bias, s = colscale, r = residual, ref computed in float64):
    |out - ref| <= 1.2 * |s| * (E + 2^-23 * |y|) + 2^-20 * (|act(y) * s| + |r|)
  - E = ceil(K / 16) * 2^-24 * (|x| @ |w|^T): the products of two bf16 values are exact in fp32, so the accumulator's
    only error is the fp32 summation; E allows every k16 step of wgmma one rounding (truncating or not) of the sum of
    magnitudes.
  - 2^-23 * |y|: the fp32 rounding of acc + bias, and the absolute error of erff in GELU's 1 + erf(y / sqrt 2) (which
    cancels for y << 0, so it is not relative to the output).
  - 1.2 bounds |act'| (GELU 1.13, SiLU and quick-GELU 1.10, ReLU 1).
  - 2^-20 relative: the fp32 roundings of the activation (__expf in SiLU / quick-GELU), the scale and the residual add.
There is no max|ref| term: a wrong constant in an activation (tanh-form GELU, quick-GELU's 1.702) or a column that
misses its bias / scale / residual is far outside it.  The worst err / bound over all cases of test 1 is 0.15 (NVIDIA
H100 80GB HBM3, 700 W power limit); `pytest -rP` prints it per case.
"""
import functools
import itertools
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from visionllm_b200 import _lib  # noqa: E402

TILES = {"1": _lib.GEMM_DEFAULT, "2": _lib.GEMM_WIDE_TILE}     # tile width in 128-column units
SENTINEL = 4320.0                                              # exact in bf16 and fp32; the kernel never writes it here


def ops():
    from visionllm_b200 import ops as o
    return o


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


ACT_REF = {                                    # float64 definitions of the fused activations
    "none": lambda y: y,
    "gelu": lambda y: 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0))),
    "relu": torch.relu,
    "silu": lambda y: y * torch.sigmoid(y),
    "quick_gelu": lambda y: y * torch.sigmoid(1.702 * y),
}


def acc_bound(x, w):
    """E: the bound of the fp32 accumulation of x @ w^T (see the module docstring)."""
    return math.ceil(x.shape[1] / 16) * 2.0 ** -24 * (x.double().abs() @ w.double().abs().T)


def padded(rows, cols, dtype, view_fill, pad_fill=SENTINEL):
    """A [rows + 1, ld] buffer (ld > cols, 16-byte row pitch) filled with pad_fill, and its top-left [rows, cols] view
    filled with view_fill."""
    per16 = 16 // torch.tensor([], dtype=dtype).element_size()
    ld = (cols + per16) // per16 * per16
    buf = torch.full((rows + 1, ld), pad_fill, dtype=dtype, device="cuda")
    view = buf[:rows, :cols]
    view.fill_(view_fill)
    return buf, view


def run_linear(x, w, n_out, out_dtype, what, **kw):
    """ops.linear into a NaN-filled [M, n_out] view of a sentinel-filled buffer: checks that every element of the view
    was written and nothing around it was."""
    M = x.shape[0]
    buf, out = padded(M, n_out, out_dtype, float("nan"))
    ops().linear(x, w, out=out, **kw)
    outside = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    outside[:M, :n_out] = False
    assert not out.isnan().any(), f"{what}: {int(out.isnan().sum())} elements of the output were never written"
    assert (buf[outside] == SENTINEL).all(), f"{what}: a store landed outside [M, n_out]"
    return out


def vector(n, gen, scale, offset=0.0):
    """A contiguous bf16 [n] vector followed by NaN in memory: a read past its end poisons the result."""
    buf = torch.full((n + 8,), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:n] = torch.randn(n, device="cuda", generator=gen) * scale + offset
    return buf[:n]


def operands(M, N, K, seed):
    """x in [-8, 8] and w such that acc + bias reaches past +-10: every activation reaches its tails."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.rand(M, K, device="cuda", generator=g) * 16 - 8).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * (0.65 / K ** 0.5)).bfloat16()
    return g, x, w


# ---------------------------------------------------------------------------------------------------------------------
# 1. the epilogue matrix against fp64
# ---------------------------------------------------------------------------------------------------------------------
# (1, 13, 64): one row, odd N inside one chunk; (77, 200, 72): ragged rows, a ragged last chunk, K past one k-block;
# (129, 4, 16): a quarter of one k-block, a single ragged row; (300, 257, 136): odd N one past a tile edge;
# (1100, 2000, 200): nine row-blocks (a second raster group of one) and more tiles than SMs.
EPI_SHAPES = [(1, 13, 64), (77, 200, 72), (129, 4, 16), (300, 257, 136), (1100, 2000, 200)]


@functools.lru_cache(maxsize=None)
def epi_problem(M, N, K):
    g, x, w = operands(M, N, K, seed=M * 7 + N)
    keep = torch.rand(M, device="cuda", generator=g) > 0.35
    keep[0] = False                                     # at least one masked row ...
    if M > 1:
        keep[-1] = True                                 # ... and one kept row
    x_poison = x.clone()                                # masked rows carry NaN and +-Inf: row_keep must still store 0
    masked = (~keep).nonzero().flatten()
    x_poison[masked, 0] = float("nan")
    x_poison[masked, 1::3] = float("inf")
    x_poison[masked, 2::3] = float("-inf")
    bias = vector(N, g, 1.5)
    scale = vector(N, g, 0.7)
    _, res = padded(M, N, torch.bfloat16, 0.0, pad_fill=float("nan"))     # ldr > n_out, NaN past each row
    res.copy_(torch.randn(M, N, device="cuda", generator=g) * 4)
    return dict(x=x, x_poison=x_poison, w=w, keep=keep, bias=bias, scale=scale, res=res,
                acc=x.double() @ w.double().T, E=acc_bound(x, w))


@pytest.mark.parametrize("act", list(ACT_REF))
@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("M,N,K", EPI_SHAPES)
def test_epilogue_matrix_vs_fp64(M, N, K, tile, act):
    """All 16 on/off combinations of bias / colscale / residual / row_keep: fp32 output within the bound of the module
    docstring of the fp64 reference, bf16 output == the fp32 output rounded, masked rows exact +0.0 (NaN / Inf input),
    kept rows identical to the unmasked call."""
    p = epi_problem(M, N, K)
    worst = 0.0
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for use_bias, use_scale, use_res in itertools.product((False, True), repeat=3):
            kw = dict(act=act, bias=p["bias"] if use_bias else None, colscale=p["scale"] if use_scale else None,
                      residual=p["res"] if use_res else None)
            y = p["acc"] + p["bias"].double() if use_bias else p["acc"]
            a = ACT_REF[act](y)
            s = p["scale"].double() if use_scale else torch.ones((), dtype=torch.float64, device="cuda")
            r = p["res"].double() if use_res else torch.zeros((), dtype=torch.float64, device="cuda")
            ref = a * s + r
            bound = 1.2 * s.abs() * (p["E"] + 2.0 ** -23 * y.abs()) + 2.0 ** -20 * ((a * s).abs() + r.abs())
            plain = None
            for use_keep in (False, True):
                what = (f"act={act} bias={use_bias} colscale={use_scale} residual={use_res} row_keep={use_keep} "
                        f"tile={tile}")
                x = p["x_poison"] if use_keep else p["x"]
                rk = p["keep"] if use_keep else None
                o32 = run_linear(x, p["w"], N, torch.float32, what, row_keep=rk, **kw)
                o16 = run_linear(x, p["w"], N, torch.bfloat16, what, row_keep=rk, **kw)
                assert same_bits(o16, o32.to(torch.bfloat16)), \
                    f"{what}: bf16 output != fp32 output rounded to bf16 ({int((bits(o16) != bits(o32.bfloat16())).sum())} elements)"
                if not use_keep:
                    err = (o32.double() - ref).abs()
                    ratio = err / bound
                    i = int(ratio.argmax())
                    worst = max(worst, float(ratio.flatten()[i]))
                    assert (err <= bound).all(), (
                        f"{what}: {int((err > bound).sum())} / {err.numel()} outside the bound; worst at "
                        f"{divmod(i, N)}: out {o32.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r} "
                        f"bound {bound.flatten()[i].item():.3g}")
                    plain = (o32, o16)
                else:
                    keep = p["keep"]
                    assert (bits(o32[~keep]) == 0).all() and (bits(o16[~keep]) == 0).all(), \
                        f"{what}: a masked row is not exact +0.0"
                    assert same_bits(o32[keep], plain[0][keep]) and same_bits(o16[keep], plain[1][keep]), \
                        f"{what}: kept rows differ from the call without row_keep"
    print(f"worst err/bound {worst:.4f}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. SwiGLU (bf16 output only; fp32 output and colscale are rejected, see tests/test_gemm_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("I", [13, 1375])
def test_swiglu_vs_fp64(I, tile):
    """Interleaved (gate, up) rows, bias on / off x residual on / off, odd I with 2I not a multiple of 64 and a ragged
    row tile: silu(gate) * up + residual within one bf16 rounding of the fp64 reference plus the fp32 bound built from
    the gate and up bounds.  The rounding term 2^-8 * |ref| is tight by construction (a bf16 rounding reaches
    2^-8 / (1 + 2^-8) of the value just above a power of two), so the margin lives in the fp32 term."""
    M, K = 200, 96
    g, x, w = operands(M, 2 * I, K, seed=I)
    bias = vector(2 * I, g, 1.5)
    _, res = padded(M, I, torch.bfloat16, 0.0, pad_fill=float("nan"))
    res.copy_(torch.randn(M, I, device="cuda", generator=g) * 4)
    acc = x.double() @ w.double().T
    E = acc_bound(x, w)
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for use_bias, use_res in itertools.product((False, True), repeat=2):
            what = f"swiglu I={I} bias={use_bias} residual={use_res} tile={tile}"
            out = run_linear(x, w, I, torch.bfloat16, what, act="swiglu", bias=bias if use_bias else None,
                             residual=res if use_res else None)
            y = acc + bias.double() if use_bias else acc
            gate, up = y[:, 0::2], y[:, 1::2]
            eg = E[:, 0::2] + 2.0 ** -23 * gate.abs()
            eu = E[:, 1::2] + 2.0 ** -23 * up.abs()
            sg = gate * torch.sigmoid(gate)
            r = res.double() if use_res else torch.zeros((), dtype=torch.float64, device="cuda")
            ref = sg * up + r
            e32 = 1.2 * eg * (up.abs() + eu) + sg.abs() * eu + 2.0 ** -20 * ((sg * up).abs() + r.abs())
            bound = 2.0 ** -8 * ref.abs() + 1.2 * e32
            err = (out.double() - ref).abs()
            assert (err <= bound).all(), \
                f"{what}: {int((err > bound).sum())} / {err.numel()} off; max err/bound {(err / bound).max().item():.3g}"


# ---------------------------------------------------------------------------------------------------------------------
# 3. schedule invariances: bit-identical, no tolerance
# ---------------------------------------------------------------------------------------------------------------------
SCHED_SHAPES = [(1100, 2000, 200), (1025, 3200, 640)]


def sched_problem(M, N, K):
    g, x, w = operands(M, N, K, seed=K)
    bias = vector(N, g, 1.5)
    res = (torch.randn(M, N, device="cuda", generator=g) * 4).bfloat16()
    return x, w, bias, res


def gelu_linear(x, w, bias, res, out_dtype):
    return ops().linear(x, w, bias=bias, act="gelu", residual=res, out_dtype=out_dtype)


@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("M,N,K", SCHED_SHAPES)
def test_sm_budget_and_slicing_are_bit_identical(M, N, K, tile):
    """Bias + GELU + residual: an SM budget of 1 / 2 / 7 / 66 CTAs (one persistent CTA walks many tiles and carries
    its stage ring and bias / scale staging across them) and row / column slices of the operands give the bytes of the
    full default launch.  The column slice starts and ends off a 64-column chunk boundary, so a chunk that is staged
    in one call is a fragment-path chunk in the other."""
    x, w, bias, res = sched_problem(M, N, K)
    r0, r1, c0, c1 = 200, M - 3, 136, 1000
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for dt in (torch.bfloat16, torch.float32):
            full = gelu_linear(x, w, bias, res, dt)
            for n in (1, 2, 7, 66):
                with _lib.knob("gemm_set_sm_limit", n, 0):
                    got = gelu_linear(x, w, bias, res, dt)
                assert same_bits(got, full), f"{dt} SM budget {n} differs from the default grid"
            rows = gelu_linear(x[r0:r1], w, bias, res[r0:r1], dt)
            assert same_bits(rows, full[r0:r1]), f"{dt} rows {r0}:{r1} differ from the full call"
            cols = gelu_linear(x, w[c0:c1], bias[c0:c1], res[:, c0:c1], dt)
            assert same_bits(cols, full[:, c0:c1]), f"{dt} columns {c0}:{c1} differ from the full call"


@pytest.mark.parametrize("M,N,K", SCHED_SHAPES)
def test_tile_widths_are_bit_identical(M, N, K):
    """128- and 256-column tiles issue the same m64n128k16 MMAs per 128 columns in the same K order and run the same
    epilogue: the same bytes, fp32 and bf16."""
    x, w, bias, res = sched_problem(M, N, K)
    for dt in (torch.bfloat16, torch.float32):
        out = {}
        for t, v in TILES.items():
            with _lib.knob("gemm_set_variant", v):
                out[t] = gelu_linear(x, w, bias, res, dt)
        assert same_bits(out["1"], out["2"]), f"{dt}: 128- and 256-column tiles differ"


# ---------------------------------------------------------------------------------------------------------------------
# 4. the other entry points of the same kernel
# ---------------------------------------------------------------------------------------------------------------------
def gemm_batched(*args, **kw):
    from visionllm_b200.train import gemm_batched as gb
    return gb(*args, **kw)


def stacked(n, rows, cols, g, scale=1.0):
    return (torch.randn(n * rows, cols, device="cuda", generator=g) * scale).bfloat16()


@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_batched_equals_separate_gemm_tn(a_mn, b_mn, tile):
    """vllm_gemm_bf16_batched (causal 0) == one vllm_gemm_bf16_tn per matrix, bit for bit, ragged N, every operand
    layout (K-major [rows, K] or MN-major [K, rows] stacks)."""
    nb, M, N = 3, 256, 200
    K = 192 if (a_mn or b_mn) else 200                  # MN-major stacks need K % 64 == 0
    g = torch.Generator(device="cuda").manual_seed(17 + 2 * a_mn + b_mn)
    A = stacked(nb, K, M, g) if a_mn else stacked(nb, M, K, g)
    B = stacked(nb, K, N, g) if b_mn else stacked(nb, N, K, g)
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for dt in (torch.bfloat16, torch.float32):
            C = gemm_batched(A, B, nb, M, N, K, a_mn=bool(a_mn), b_mn=bool(b_mn), out_dtype=dt)
            for b in range(nb):
                Ab = A[b * K:(b + 1) * K] if a_mn else A[b * M:(b + 1) * M]
                Bb = B[b * K:(b + 1) * K] if b_mn else B[b * N:(b + 1) * N]
                Cb = ops().gemm_tn(Ab, Bb, a_mn=bool(a_mn), b_mn=bool(b_mn), out_dtype=dt)
                assert same_bits(C[b * M:(b + 1) * M], Cb), f"{dt} matrix {b} differs from its own gemm_tn call"


@pytest.mark.parametrize("tile", list(TILES))
def test_batched_causal_modes_match_mode0(tile):
    """Causal modes 2 / 3 skip k-blocks where the operand is exactly zero (A(m, k) = 0 for k < m / k > m): the result
    equals mode 0 bit for bit, every operand layout.  Mode 1 skips output tiles strictly above the diagonal: those keep
    what the buffer held, every other element equals mode 0."""
    nb, T, N = 3, 512, 200
    g = torch.Generator(device="cuda").manual_seed(23)
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for mode in (2, 3):
            a = torch.randn(nb, T, T, device="cuda", generator=g).bfloat16()           # A(m, k) per matrix
            a = a.triu() if mode == 2 else a.tril()
            b = torch.randn(nb, N, T, device="cuda", generator=g).bfloat16()           # B(n, k)
            for a_mn, b_mn in itertools.product((False, True), repeat=2):
                A = (a.transpose(1, 2) if a_mn else a).contiguous().view(nb * T, T)
                B = (b.transpose(1, 2) if b_mn else b).contiguous().view(-1, N if b_mn else T)
                for dt in (torch.bfloat16, torch.float32):
                    full = gemm_batched(A, B, nb, T, N, T, a_mn=a_mn, b_mn=b_mn, out_dtype=dt)
                    cut = gemm_batched(A, B, nb, T, N, T, a_mn=a_mn, b_mn=b_mn, causal=mode, out_dtype=dt)
                    assert same_bits(cut, full), f"causal {mode} a_mn={a_mn} b_mn={b_mn} {dt} differs from mode 0"
        q, k = stacked(nb, T, 128, g), stacked(nb, T, 128, g)
        bn = 128 * int(tile)
        m_loc = torch.arange(nb * T, device="cuda") % T
        n = torch.arange(T, device="cuda")
        skipped = (n // bn * bn)[None, :] >= (m_loc // 128 * 128)[:, None] + 128     # tile's first column > its last row
        assert skipped.any()
        for dt in (torch.bfloat16, torch.float32):
            full = gemm_batched(q, k, nb, T, T, 128, out_dtype=dt)
            out = torch.full((nb * T, T), SENTINEL, dtype=dt, device="cuda")
            gemm_batched(q, k, nb, T, T, 128, causal=1, out_dtype=dt, out=out)
            assert (out[skipped] == SENTINEL).all(), f"causal 1 {dt} wrote a tile above the diagonal"
            assert same_bits(out[~skipped], full[~skipped]), f"causal 1 {dt} differs from mode 0 on or below the diagonal"


@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("B,H,W,C,Cout,k,act", [(2, 13, 17, 64, 200, 3, "relu"), (1, 9, 30, 128, 72, 3, "gelu"),
                                                 (1, 12, 11, 64, 96, 5, None)])
def test_conv_rows_equals_linear_on_im2col(B, H, W, C, Cout, k, act, tile):
    """vllm_conv_rows_bf16 (implicit GEMM over the zero-padded map) == ops.linear on an explicit im2col in (dy, dx, c)
    order, bit for bit on the rows inside an image: a kernel row segment is whole k-blocks (k * C % 64 == 0), so both
    sum the same products in the same order."""
    p = k // 2
    g = torch.Generator(device="cuda").manual_seed(B * 100 + C + k)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, k * k * C, device="cuda", generator=g) / (k * k * C) ** 0.5).bfloat16()
    bias = torch.randn(Cout, device="cuda", generator=g).bfloat16()
    xp = torch.nn.functional.pad(x, (0, 0, p, p, p, p))
    cols = xp.unfold(1, k, 1).unfold(2, k, 1)                            # [B, H, W, C, dy, dx]
    cols = cols.permute(0, 1, 2, 4, 5, 3).reshape(B * H * W, k * k * C).contiguous()
    with _lib.knob("gemm_set_variant", TILES[tile]):
        got = ops().conv2d_s1_rows(x, w, bias, k, p, act=act)
        ref = ops().linear(cols, w, bias=bias, act=act).view(B, H, W, Cout)
    assert same_bits(got.contiguous(), ref)
