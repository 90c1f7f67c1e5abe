"""GPU: the row kernels of the training step (csrc/train_ops.cu, visionllm_b200/train.py) against float64 references of
the same ops on the same bf16 / fp32 inputs, with exact probes, bit-identities and NaN sentinels around every output.

Kernels: RMSNorm backward (per-CTA dweight partials), the causal softmax and its backward, SwiGLU forward / backward,
the CE loss and `CrossEntropyFn`, RoPE backward (`RopeFn`, `QKVRopeFn`) and the head stacking of the attention backward.

The checker is `rounds` of tests/bf16_rounding.py: away from a bf16 rounding midpoint within E of the float64 value z,
the bf16 output is RN_bf16(z) bit for bit.  u = 2^-24; no bound has a max|ref| term.  Bounds, per kernel:
  RMSNorm bwd   d = 8 VPT + 13 (per-thread chain, warp tree, 8-warp sum); r = 1 / sqrt(mean(x^2) + eps) carries
                er = (d / 2 + 6) u (the sum of squares, the division, rsqrtf's 2 ulp).  With a = dy w, n = x r,
                m = mean(a n):  dx = r (a - n m) within 1.25 r (|a - n m| (er + 3u) + |n| (|m| (2 er + 4u) + dm)),
                dm = (er + (d + 3) u) mean|a n| + u |m| -- an absolute term for the cancellation in the bracket.
                dw = sum_rows dy RN_bf16(n): where RN_bf16(n) has two candidates within (er + u)|n| the row may use either
                (sum of |dy| |hi - lo| over those ties), plus the fp32 chain c u sum |dy| max(|lo|, |hi|) with
                c = rows_per_cta + ceil(n_partials / 8) + 8.
  softmax       P = softmax(s S) over keys <= query, s the fp32 scale:  E_j = 1.25 P_j (e_j + max_k e_k + (d + 3) u),
                e_j = 2^-21 + |x_j| 2^-23 + u (|s S_j| + |max| + |x_j|), x_j = s S_j - max (__expf of an fp32 argument).
  softmax bwd   dS = s P (dP - sum P dP):  E = 1.25 s |P| (d u sum |P dP| + 3u |dP - sum P dP|).
  SwiGLU        sigmoid through __expf: delta_s = s ((1 - s)(2^-21 + |g| 2^-23) + min(2u, 2 (1 - s))), plus s itself
                where s < 2^-125 (exp overflows to inf, the kernel's s is 0).  h = g s u within |g u| (delta_s + 2u s);
                du = dh g s within |dh g| (delta_s + u s); dg = dh u s b, b = 1 + g (1 - s), within
                1.25 |dh u| (delta_s |b| + s delta_b + 2u s |b|), delta_b = |g| (delta_s + u (1 - s)) + u |g (1 - s)| + u |b|
                -- absolute in b, which cancels at g = -1.278.
  CE loss       per row  dlse = (ceil(V / 512) + 21) u + mean_p(4u + u |l - max|) + 2u |log sum| + u |lse|;
                loss within (sum_rows (dlse + u loss_r) + n u sum_rows loss_r) / n + u loss (the atomic row sum).
                dlogits = (p - onehot) / n within 1.25 (p (dlse + u |l - lse| + 4u) + 3u |p - onehot|) / n + 2^-140 / n.
  dloss scale   c dlogits within two bf16 roundings of c (p - onehot) / n; mean signed relative error <= 2^-12.
  RoPE bwd      bit-identical to torch autograd of the HF bf16 formula q cos + rotate_half(q) sin.

`pytest -s` prints the worst observed err / E per family.  On an NVIDIA H100 80GB HBM3 at 700 W the values are listed
in DESIGN.md section 4.
"""
import math

import numpy as np
import pytest
import torch

from visionllm_b200 import _lib
from bf16_rounding import U, bf16_ulp, note_ratio, print_report, rn_bf16, rounds, within

pytestmark = pytest.mark.gpu
EINVAL, EUNSUPPORTED, EALIGN = -1, -2, -3
NAN = float("nan")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("training kernels")


# ---------------------------------------------------------------------------------------------------------------------
# buffers
# ---------------------------------------------------------------------------------------------------------------------
def stream():
    return torch.cuda.current_stream().cuda_stream


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def pitched(data, ld, fill=NAN):
    """A [rows, ld] buffer filled with `fill` holding `data` [rows, cols] in its first columns, and that view."""
    rows, cols = data.shape
    buf = torch.full((rows, ld), fill, dtype=data.dtype, device="cuda")
    buf[:, :cols] = data
    return buf, buf[:, :cols]


class Out:
    """A [rows, cols] output view with row pitch ld inside a buffer of `fill` with a spare row above and below.
    `check()` asserts every element of the view was written and nothing around it changed."""

    def __init__(self, rows, cols, ld=None, dtype=torch.bfloat16, fill=NAN):
        ld = ld or cols
        self.buf = torch.full((rows + 2, ld), NAN, dtype=dtype, device="cuda")
        self.buf[1:rows + 1, :cols] = fill
        self.view = self.buf[1:rows + 1, :cols]
        self.before = bits(self.buf).clone()
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[1:rows + 1, :cols] = True

    def untouched(self):
        return torch.equal(bits(self.buf), self.before)

    def check(self, what):
        assert not self.view.isnan().any(), f"{what}: {int(self.view.isnan().sum())} output elements never written"
        assert torch.equal(bits(self.buf)[~self.inside], self.before[~self.inside]), f"{what}: a store landed outside"
        return self.view


def vector(values):
    """A contiguous copy of `values` followed by NaN in memory: a read past its end poisons the result."""
    n = values.numel()
    buf = torch.full((n + 8,), NAN, dtype=values.dtype, device="cuda")
    buf[:n] = values.flatten()
    return buf[:n]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def f32(v):
    return float(np.float32(v))


def vpt(n_cols):
    nvec = n_cols // 8
    return 1 if nvec <= 256 else (2 if nvec <= 512 else 4)


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm backward
# ---------------------------------------------------------------------------------------------------------------------
def rms_bwd(x, w, dy, dx, dw, part, n_part, eps=1e-6):
    rows, cols = x.shape
    return _lib.lib().vllm_rmsnorm_bwd_ws_bf16(x.data_ptr(), x.stride(0), w.data_ptr(), dy.data_ptr(), dy.stride(0),
                                               dx.data_ptr(), dx.stride(0), dw.data_ptr(), part.data_ptr(), n_part, rows,
                                               cols, eps, stream())


def rms_plan(rows):
    """(CTAs = partial rows, rows per CTA) of the backward launch, from the library's own workspace query."""
    n = _lib.lib().vllm_rmsnorm_bwd_partials(rows)
    return n, -(-rows // n)


def rows_one_per_cta():
    """The largest row count the backward still spreads one row per CTA."""
    P = _lib.lib().vllm_rmsnorm_bwd_partials
    lo, hi = 1, 1 << 22
    assert P(lo) == lo and P(hi) < hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if P(mid) == mid else (lo, mid)
    return lo


def rms_inputs(kind, rows, cols, g):
    x = torch.randn(rows, cols, device="cuda", generator=g)
    if kind == "offset":
        x = x + 30.0
    elif kind == "outlier":
        ch = torch.randperm(cols, device="cuda", generator=g)[:max(1, cols // 512)]
        x[:, ch] *= 300.0
    elif kind == "tiny":                                  # mean(x^2) ~ 1e-10, far below eps = 1e-6
        x = x * 1e-5
    dy = (torch.randn(rows, cols, device="cuda", generator=g) * 0.5).bfloat16()
    return x.bfloat16(), dy


def rms_bwd_ref(x, w, dy, eps):
    """(z_dx, E_dx, n, E_n) of the bounds in the module docstring."""
    cols = x.shape[1]
    d = 8 * vpt(cols) + 13
    xd, wd, gd = x.double(), w.double(), dy.double()
    r = 1.0 / torch.sqrt((xd * xd).mean(-1, keepdim=True) + f32(eps))
    n = xd * r
    a = gd * wd
    m = (a * n).mean(-1, keepdim=True)
    br = a - n * m
    er = (d / 2 + 6) * U
    dm = (er + (d + 3) * U) * (a * n).abs().mean(-1, keepdim=True) + U * m.abs()
    E = 1.25 * r * (br.abs() * (er + 3 * U) + n.abs() * (m.abs() * (2 * er + 4 * U) + dm))
    return r * br, E, n, (er + U) * n.abs()


def check_dw(dw, dy, n, En, chain, family, what):
    lo, hi = rn_bf16(n - En), rn_bf16(n + En)
    gd = dy.double()
    z = (gd * rn_bf16(n)).sum(0)
    E = (gd.abs() * (hi - lo)).sum(0) + chain * U * (gd.abs() * torch.maximum(lo.abs(), hi.abs())).sum(0)
    within(dw, z, E, family, what)


RMS_COLS = [8, 2048, 2056, 4096, 4104, 5120, 6144, 8192]


@pytest.mark.parametrize("kind", ["normal", "offset", "outlier", "tiny"])
@pytest.mark.parametrize("cols", RMS_COLS)
def test_rmsnorm_backward_vs_fp64(cols, kind):
    """dx and dw against fp64 at 1 row, the most rows that still give one row per CTA, one more (two per CTA) and 8192
    rows; inputs and dy in pitched views with NaN in the gap, NaN after w, dx inside a NaN sentinel and a NaN-prefilled
    dw.  Bit-identical across runs and pitches."""
    g = gen(cols * 5 + len(kind))
    eps = 1e-6
    r1 = rows_one_per_cta()
    w = vector((1 + 0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16())
    for rows in (1, r1, r1 + 1, 8192):
        n_ctas, rpc = rms_plan(rows)
        assert (rpc == 1) == (rows <= r1)
        x, dy = rms_inputs(kind, rows, cols, g)
        _, xv = pitched(x, cols + 24)
        _, gv = pitched(dy, cols + 40)
        part = torch.full((n_ctas, cols), NAN, device="cuda")
        dx, dw = Out(rows, cols, cols + 16), Out(1, cols, dtype=torch.float32)
        assert rms_bwd(xv, w, gv, dx.view, dw.view[0], part, n_ctas, eps) == 0
        torch.cuda.synchronize()
        what = f"rows={rows} cols={cols} {kind}"
        y, yw = dx.check("dx " + what), dw.check("dw " + what)[0]
        z, E, n, En = rms_bwd_ref(x, w, dy, eps)
        rounds(y, z, E, "rmsnorm_bwd_dx", what)
        check_dw(yw, dy, n, En, rpc + -(-n_ctas // 8) + 8, "rmsnorm_bwd_dw", what)
        # bit-identities: a second run, contiguous views (another pitch), a larger workspace
        dx2, dw2 = torch.empty_like(x), torch.empty(cols, device="cuda")
        part2 = torch.empty((n_ctas + 3, cols), device="cuda")
        assert rms_bwd(x, w, dy, dx2, dw2, part2, n_ctas + 3, eps) == 0
        assert same_bits(dx2, y) and same_bits(dw2, yw), f"partials form not reproducible across pitches: {what}"


def test_rmsnorm_backward_probes():
    """dy = 0 gives exact zeros in dx and dw; rows of a CTA group with dy = 0 add nothing to dw."""
    g = gen(11)
    for cols in (8, 4104, 8192):
        rows = rows_one_per_cta() + 1
        n_ctas, _ = rms_plan(rows)
        x, _ = rms_inputs("outlier", rows, cols, g)
        w = vector((1 + 0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16())
        dy = torch.zeros(rows, cols, dtype=torch.bfloat16, device="cuda")
        part = torch.full((n_ctas, cols), NAN, device="cuda")
        dx, dw = Out(rows, cols), Out(1, cols, dtype=torch.float32)
        assert rms_bwd(x, w, dy, dx.view, dw.view[0], part, n_ctas) == 0
        torch.cuda.synchronize()
        assert (dx.check("dx") == 0).all() and (dw.check("dw") == 0).all(), f"dy = 0 is not exact 0 at cols={cols}"


def test_rmsnorm_backward_rejections_leave_outputs_untouched():
    L = _lib.lib()
    st = stream()
    x = torch.randn(16, 8208, device="cuda").bfloat16()
    w = torch.ones(8208, device="cuda").bfloat16()
    dx, dw = Out(4, 8208), Out(1, 8208, dtype=torch.float32)
    part = torch.full((64, 8208), NAN, device="cuda")
    xp, wp, dxp, dwp, pp = x.data_ptr(), w.data_ptr(), dx.view.data_ptr(), dw.view.data_ptr(), part.data_ptr()
    lx, ld = x.stride(0), dx.view.stride(0)
    n_ok = L.vllm_rmsnorm_bwd_partials(4)
    cases = {   # (x, ldx, dy, ldy, dx, lddx, cols, n_partials, expected)
        "cols % 8": (xp, lx, xp, lx, dxp, ld, 100, n_ok, EINVAL),
        "cols > 8192": (xp, lx, xp, lx, dxp, ld, 8200, n_ok, EUNSUPPORTED),
        "x misaligned": (xp + 2, lx, xp, lx, dxp, ld, 256, n_ok, EALIGN),
        "dy misaligned": (xp, lx, xp + 2, lx, dxp, ld, 256, n_ok, EALIGN),
        "dx misaligned": (xp, lx, xp, lx, dxp + 2, ld, 256, n_ok, EALIGN),
        "ldx % 8": (xp, 260, xp, lx, dxp, ld, 256, n_ok, EALIGN),
        "ldy % 8": (xp, lx, xp, 260, dxp, ld, 256, n_ok, EALIGN),
        "lddx % 8": (xp, lx, xp, lx, dxp, 260, 256, n_ok, EALIGN),
    }
    for what, (a, la, b, lb, c, lc, cols, npart, rc) in cases.items():
        assert L.vllm_rmsnorm_bwd_ws_bf16(a, la, wp, b, lb, c, lc, dwp, pp, npart, 4, cols, 1e-6, st) == rc, what
    assert L.vllm_rmsnorm_bwd_ws_bf16(xp, lx, wp, xp, lx, dxp, ld, dwp, pp, n_ok - 1, 4, 256, 1e-6, st) == EINVAL
    assert L.vllm_rmsnorm_bwd_ws_bf16(xp, lx, wp, xp, lx, dxp, ld, dwp, pp + 4, n_ok, 4, 256, 1e-6, st) == EALIGN
    torch.cuda.synchronize()
    assert dx.untouched() and dw.untouched(), "a rejected call wrote to its outputs"
    assert part.isnan().all(), "a rejected call wrote to the workspace"


# ---------------------------------------------------------------------------------------------------------------------
# causal softmax and its backward
# ---------------------------------------------------------------------------------------------------------------------
def softmax_call(s, n_mat, T, scale):
    return _lib.lib().vllm_softmax_causal_bf16(s.data_ptr(), s.stride(0), n_mat, T, scale, stream())


def ds_call(p, dp, n_mat, T, scale):
    return _lib.lib().vllm_attn_ds_bf16(p.data_ptr(), dp.data_ptr(), p.stride(0), n_mat, T, scale, stream())


def regions(T, ld):
    """Masks over a [T, ld] matrix: `low` (j <= i), `zero` (above the diagonal inside the row's 256-aligned diagonal
    block: the kernels write exact 0 there), `keep` (beyond that block and the pitch gap: never written)."""
    i = torch.arange(T, device="cuda")[:, None]
    j = torch.arange(ld, device="cuda")[None, :]
    end = torch.clamp((i // 256 + 1) * 256, max=T)
    return j <= i, (j > i) & (j < end), j >= end


def causal_stack(vals, T, ld, low):
    """[n_mat * T, ld] bf16 holding vals on and below the diagonal and NaN everywhere else."""
    n_mat = vals.shape[0]
    buf = torch.full((n_mat, T, ld), NAN, dtype=torch.bfloat16, device="cuda")
    buf[:, :, :T] = torch.where(low[:, :T], vals, torch.full_like(vals, NAN))
    return buf.view(n_mat * T, ld)


def check_regions(out, before, n_mat, T, ld, zero, keep, what):
    o = out.view(n_mat, T, ld)
    assert (o[:, zero] == 0).all(), f"{what}: not exact 0 above the diagonal inside the diagonal block"
    assert torch.equal(bits(o)[:, keep], bits(before.view(n_mat, T, ld))[:, keep]), f"{what}: wrote beyond the diagonal block"


SOFTMAX_T = [256, 2048, 2304, 4096, 4352, 8192]


@pytest.mark.parametrize("T", SOFTMAX_T)
def test_causal_softmax_and_backward_vs_fp64(T):
    """P and dS against fp64 at both scales, several matrices, ld > T; NaN above the diagonal of S and dP and in the
    pitch gap: exact 0 inside the diagonal block, NaN untouched beyond it, no NaN in a valid element."""
    g = gen(T)
    n_mat = 2 if T > 4096 else 3
    ld = T + 16
    low, zero, keep = regions(T, ld)
    lowT = low[:, :T]
    d = 8 * vpt(T) + 13
    for scale in (0.125, 128 ** -0.5):
        sf = f32(scale)
        vals = (torch.randn(n_mat, T, T, device="cuda", generator=g) * 4).bfloat16()
        s = causal_stack(vals, T, ld, low)
        before = s.clone()
        assert softmax_call(s, n_mat, T, scale) == 0
        torch.cuda.synchronize()
        what = f"T={T} scale={scale}"
        check_regions(s, before, n_mat, T, ld, zero, keep, "softmax " + what)
        p = s.view(n_mat, T, ld)[:, :, :T]
        assert not p[:, lowT].isnan().any(), f"softmax {what}: NaN reached a valid element"
        v = torch.where(lowT, vals.double() * sf, torch.full((), -math.inf, dtype=torch.float64, device="cuda"))
        mx = v.amax(-1, keepdim=True)
        x = v - mx
        z = torch.softmax(v, -1)
        e = 2.0 ** -21 + x.abs() * 2.0 ** -23 + U * (v.abs() + mx.abs() + x.abs())
        e = torch.where(lowT, e, torch.zeros_like(e))
        E = 1.25 * z * (e + e.amax(-1, keepdim=True) + (d + 3) * U)
        rounds(p[:, lowT], z[:, lowT], E[:, lowT], "softmax_causal", what)
        del v, x, e, E
        # backward on this P (NaN beyond the diagonal block) and a dP with NaN above the diagonal
        dvals = (torch.randn(n_mat, T, T, device="cuda", generator=g) * 2).bfloat16()
        dp = causal_stack(dvals, T, ld, low)
        before = dp.clone()
        assert ds_call(s, dp, n_mat, T, scale) == 0
        torch.cuda.synchronize()
        check_regions(dp, before, n_mat, T, ld, zero, keep, "attn_ds " + what)
        ds = dp.view(n_mat, T, ld)[:, :, :T]
        assert not ds[:, lowT].isnan().any(), f"attn_ds {what}: NaN reached a valid element"
        pd = torch.where(lowT, p.double(), torch.zeros((), dtype=torch.float64, device="cuda"))
        gd = torch.where(lowT, dvals.double(), torch.zeros((), dtype=torch.float64, device="cuda"))
        dot = (pd * gd).sum(-1, keepdim=True)
        z = sf * pd * (gd - dot)
        E = 1.25 * sf * pd.abs() * (d * U * (pd * gd).abs().sum(-1, keepdim=True) + 3 * U * (gd - dot).abs())
        rounds(ds[:, lowT], z[:, lowT], E[:, lowT], "softmax_bwd", what)


@pytest.mark.parametrize("T", SOFTMAX_T)
def test_causal_softmax_exact_probes(T):
    """Key count: a constant row gives P[i, j] = RN_bf16(fl32(1 / (i + 1))) for every j <= i, bit for bit.  Power-of-two
    P with small-integer dP at scale 1/8 gives dS exactly."""
    g = gen(T + 1)
    n_mat, ld = 2, T + 8
    low, zero, keep = regions(T, ld)
    lowT = low[:, :T]
    s = causal_stack(torch.full((n_mat, T, T), 0.75, dtype=torch.bfloat16, device="cuda"), T, ld, low)
    before = s.clone()
    assert softmax_call(s, n_mat, T, 128 ** -0.5) == 0
    torch.cuda.synchronize()
    check_regions(s, before, n_mat, T, ld, zero, keep, f"key-count probe T={T}")
    inv = torch.from_numpy(np.float32(1) / np.arange(1, T + 1, dtype=np.float32)).cuda().double()
    want = rn_bf16(inv)[:, None].expand(T, T)
    p = s.view(n_mat, T, ld)[:, :, :T]
    assert torch.equal(p.double()[:, lowT], want[lowT].expand(n_mat, -1)), f"key-count probe T={T}: P != bf16(1/(i+1))"
    # dS exact: P = 2^-k (k < 7), dP in -3..3, scale 1/8
    pv = torch.exp2(-torch.randint(0, 7, (n_mat, T, T), device="cuda", generator=g).double()).bfloat16()
    dv = torch.randint(-3, 4, (n_mat, T, T), device="cuda", generator=g).bfloat16()
    pp, dp = causal_stack(pv, T, ld, low), causal_stack(dv, T, ld, low)
    before = dp.clone()
    assert ds_call(pp, dp, n_mat, T, 0.125) == 0
    torch.cuda.synchronize()
    check_regions(dp, before, n_mat, T, ld, zero, keep, f"dS probe T={T}")
    pd = torch.where(lowT, pv.double(), torch.zeros((), dtype=torch.float64, device="cuda"))
    gd = torch.where(lowT, dv.double(), torch.zeros((), dtype=torch.float64, device="cuda"))
    z = 0.125 * pd * (gd - (pd * gd).sum(-1, keepdim=True))
    ds = dp.view(n_mat, T, ld)[:, :, :T].double()
    assert torch.equal(ds[:, lowT], rn_bf16(z)[:, lowT]), f"dS probe T={T}: not exact"


def test_causal_softmax_rejections_leave_the_buffer_untouched():
    L = _lib.lib()
    st = stream()
    s = torch.full((512, 264), 1.0, dtype=torch.bfloat16, device="cuda")
    before = s.clone()
    sp = s.data_ptr()
    for fn in (lambda *a: L.vllm_softmax_causal_bf16(*a), lambda p, ld, n, T, sc, stm: L.vllm_attn_ds_bf16(sp, p, ld, n, T, sc, stm)):
        assert fn(sp, 264, 2, 252, 0.1, st) == EINVAL                  # T % 8
        assert fn(sp, 248, 2, 256, 0.1, st) == EINVAL                  # ld < T
        assert fn(sp, 260, 2, 256, 0.1, st) == EINVAL                  # ld % 8
        assert fn(sp + 2, 264, 2, 256, 0.1, st) == EALIGN
        assert fn(sp, 8200, 1, 8200, 0.1, st) == EUNSUPPORTED          # T > 8192
    assert L.vllm_attn_ds_bf16(sp + 2, sp, 264, 2, 256, 0.1, st) == EALIGN
    torch.cuda.synchronize()
    assert same_bits(s, before)


def rel(a, b):
    return float(torch.linalg.norm((a.double() - b.double()).flatten()) / torch.linalg.norm(b.double().flatten()))


def hf_eager_attention_grads(qkv5, do, scale, dtype):
    """d(q, k, v) of HF's eager attention (repeat_kv, scores in `dtype`, fp32 softmax cast back) by torch autograd."""
    B, T, P, nkv, D = qkv5.shape
    G = P - 2
    t = qkv5.detach().to(dtype).requires_grad_(True)
    q = t[:, :, :G].reshape(B, T, G * nkv, D).transpose(1, 2)
    k = t[:, :, G].transpose(1, 2).repeat_interleave(G, 1)
    v = t[:, :, G + 1].transpose(1, 2).repeat_interleave(G, 1)
    s = torch.matmul(q, k.transpose(2, 3)) * scale
    s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device="cuda").triu(1), torch.finfo(dtype).min)
    p = torch.softmax(s, -1, dtype=torch.float32 if dtype != torch.float64 else dtype).to(dtype)
    o = torch.matmul(p, v).transpose(1, 2).reshape(B, T, G * nkv * D)
    o.backward(do.to(dtype))
    return t.grad


@pytest.mark.parametrize("G", [1, 6])
@pytest.mark.parametrize("T", [4096, 8192])
def test_attention_backward_never_reads_the_unwritten_region(T, G):
    """attention_backward_packed replayed step by step into NaN-prefilled S / dP / gradient buffers is bit-identical to
    the production call: no causal GEMM reads the part of S or dP the causal score GEMM and the row kernels leave
    unwritten.  dq / dk / dv meet the module rule of HF's eager bf16 attention against fp64 autograd."""
    from visionllm_b200 import train as TR
    B, D = 1, 128
    nkv = 2 if G == 1 else 1
    nq = G * nkv
    g = gen(T + G)
    qkv5 = (torch.randn(B, T, G + 2, nkv, D, device="cuda", generator=g) * 0.5).bfloat16()
    do = (torch.randn(B, T, nq * D, device="cuda", generator=g) * 0.5).bfloat16()
    scale = D ** -0.5
    got = TR.attention_backward_packed(qkv5, do, scale)
    L = _lib.lib()
    BQ, BKV = B * nq, B * nkv
    stk = TR.head_stack_qkv(qkv5.reshape(B, T, -1), nq, nkv, D)
    qs, ks, vs = stk[:BQ * T], stk[BQ * T:(BQ + BKV) * T], stk[(BQ + BKV) * T:]
    dos = TR.head_stack(do, B, T, 1, nq, D, True).view(BQ * T, D)
    p = torch.full((BQ * T, T), NAN, dtype=torch.bfloat16, device="cuda")
    dp = torch.full_like(p, NAN)
    TR.gemm_batched(qs, ks, BQ, T, T, D, causal=1, group=G, out=p)
    assert softmax_call(p, BQ, T, scale) == 0
    TR.gemm_batched(dos, vs, BQ, T, T, D, causal=1, group=G, out=dp)
    assert ds_call(p, dp, BQ, T, scale) == 0
    dstk = torch.full_like(stk, NAN)
    dqs, dks, dvs = dstk[:BQ * T], dstk[BQ * T:(BQ + BKV) * T], dstk[(BQ + BKV) * T:]
    TR.gemm_batched(p, dos, BQ, T, D, T, a_mn=True, b_mn=True, causal=2, out=dvs, group=G, reduce=True)
    TR.gemm_batched(dp, qs, BQ, T, D, T, a_mn=True, b_mn=True, causal=2, out=dks, group=G, reduce=True)
    TR.gemm_batched(dp, ks, BQ, T, D, T, b_mn=True, causal=3, out=dqs, group=G)
    dqkv = torch.full((B, T, (G + 2) * nkv * D), NAN, dtype=torch.bfloat16, device="cuda")
    TR.head_stack_qkv(dqkv, nq, nkv, D, stacks=dstk)
    torch.cuda.synchronize()
    assert not dqkv.isnan().any(), "NaN from the unwritten region of S / dP reached a gradient"
    assert same_bits(dqkv.view_as(got), got), "the replay into NaN-prefilled buffers differs from the production call"
    del p, dp, dstk, stk
    ref = hf_eager_attention_grads(qkv5, do, scale, torch.float64)
    bf = hf_eager_attention_grads(qkv5, do, scale, torch.bfloat16)
    for name, sl in (("dq", slice(0, G)), ("dk", slice(G, G + 1)), ("dv", slice(G + 1, G + 2))):
        a, b = rel(got[:, :, sl], ref[:, :, sl]), rel(bf[:, :, sl], ref[:, :, sl])
        note_ratio("attention_bwd_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (name, T, G, a, b)


# ---------------------------------------------------------------------------------------------------------------------
# SwiGLU
# ---------------------------------------------------------------------------------------------------------------------
def swiglu_fwd_call(gu, h, rows, inter):
    return _lib.lib().vllm_swiglu_fwd_bf16(gu.data_ptr(), gu.stride(0), h.data_ptr(), h.stride(0), rows, inter, stream())


def swiglu_bwd_call(gu, dh, dgu, rows, inter):
    return _lib.lib().vllm_swiglu_bwd_bf16(gu.data_ptr(), gu.stride(0), dh.data_ptr(), dh.stride(0), dgu.data_ptr(),
                                           dgu.stride(0), rows, inter, stream())


def sigmoid_err(gd):
    """fp64 sigmoid and the bound of the kernel's 1 / (1 + __expf(-g)) (module docstring)."""
    s = torch.sigmoid(gd)
    oms = torch.sigmoid(-gd)                             # 1 - s without cancellation
    ee = 2.0 ** -21 + gd.abs() * 2.0 ** -23
    ds = s * (oms * ee + torch.minimum(torch.full_like(oms, 2 * U), 2 * oms))
    ds = ds + torch.where(s < 2.0 ** -125, s, torch.zeros_like(s))
    return s, oms, ds


def swiglu_gates(rows, inter, g):
    """Gates N(0, 3); every bf16 value in [-1.4, -1.15] (silu' crosses zero at -1.278) on row 0; +-60, +-80, +-100 and
    +-bf16 max on row 1, whose up and dh values stay within 1 so that the products are finite."""
    gate = torch.randn(rows, inter, device="cuda", generator=g) * 3
    up = torch.randn(rows, inter, device="cuda", generator=g)
    dense = torch.arange(-1.4, -1.15, 2.0 ** -8, device="cuda").bfloat16().unique().float()
    gate[0, :dense.numel()] = dense
    if rows > 1:
        big = float(torch.finfo(torch.bfloat16).max)
        ext = torch.tensor([60.0, -60.0, 80.0, -80.0, 100.0, -100.0, 88.5, -88.5, 89.5, -89.5, big, -big], device="cuda")
        gate[1, :ext.numel()] = ext
        up[1] = up[1].clamp(-1, 1)
    gu = torch.stack([gate, up], -1).reshape(rows, 2 * inter).bfloat16()
    dh = (torch.randn(rows, inter, device="cuda", generator=g) * 0.5).clamp(-1, 1).bfloat16()
    return gu, dh


@pytest.mark.parametrize("inter", [1376, 11008, 16384])
def test_swiglu_vs_fp64(inter):
    """Forward and backward against fp64 with enough rows that the grid-stride loop takes several passes, and 1 row;
    pitched gu / dh / outputs with NaN gaps; row slices and contiguous copies bit-identical."""
    g = gen(inter)
    threads = torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256     # the kernels' grid cap
    rows = 2 * threads * 8 // inter + 5                                                 # > 2 passes of the loop
    assert rows * inter // 8 > 2 * threads
    gu, dh = swiglu_gates(rows, inter, g)
    _, guv = pitched(gu, 2 * inter + 40)
    _, dhv = pitched(dh, inter + 8)
    h, dgu = Out(rows, inter, inter + 16), Out(rows, 2 * inter, 2 * inter + 24)
    assert swiglu_fwd_call(guv, h.view, rows, inter) == 0
    assert swiglu_bwd_call(guv, dhv, dgu.view, rows, inter) == 0
    torch.cuda.synchronize()
    y, dy = h.check("swiglu fwd"), dgu.check("swiglu bwd")
    assert y.isfinite().all() and dy.isfinite().all(), "non-finite output"
    gd, ud = gu[:, 0::2].double(), gu[:, 1::2].double()
    hd = dh.double()
    s, oms, ds = sigmoid_err(gd)
    rounds(y, gd * s * ud, (gd * ud).abs() * (ds + 2 * U * s), "swiglu_fwd", f"I={inter}")
    b = 1 + gd * oms
    db = gd.abs() * (ds + U * oms) + U * (gd * oms).abs() + U * b.abs()
    rounds(dy[:, 0::2], hd * ud * s * b, 1.25 * (hd * ud).abs() * (ds * b.abs() + s * db + 2 * U * s * b.abs()),
           "swiglu_bwd_dg", f"I={inter}")
    rounds(dy[:, 1::2], hd * gd * s, (hd * gd).abs() * (ds + U * s), "swiglu_bwd_du", f"I={inter}")
    for lo, hi in ((0, 1), (1, 2), (rows - 3, rows), (7, 40)):
        hs, dgs = Out(hi - lo, inter), Out(hi - lo, 2 * inter)
        assert swiglu_fwd_call(gu[lo:hi], hs.view, hi - lo, inter) == 0
        assert swiglu_bwd_call(gu[lo:hi], dh[lo:hi], dgs.view, hi - lo, inter) == 0
        torch.cuda.synchronize()
        assert same_bits(hs.check("slice"), y[lo:hi]) and same_bits(dgs.check("slice"), dy[lo:hi]), f"rows {lo}:{hi} differ"


def test_swiglu_rejections_leave_outputs_untouched():
    L = _lib.lib()
    st = stream()
    gu = torch.randn(4, 512, device="cuda").bfloat16()
    h, dgu = Out(4, 256), Out(4, 512)
    gp, hp, dp = gu.data_ptr(), h.view.data_ptr(), dgu.view.data_ptr()
    assert L.vllm_swiglu_fwd_bf16(gp, 512, hp, 256, 4, 252, st) == EINVAL
    assert L.vllm_swiglu_fwd_bf16(gp + 2, 512, hp, 256, 4, 256, st) == EALIGN
    assert L.vllm_swiglu_fwd_bf16(gp, 508, hp, 256, 4, 256, st) == EALIGN
    assert L.vllm_swiglu_bwd_bf16(gp, 512, gp, 256, dp, 512, 4, 252, st) == EINVAL
    assert L.vllm_swiglu_bwd_bf16(gp, 512, gp + 2, 256, dp, 512, 4, 256, st) == EALIGN
    assert L.vllm_swiglu_bwd_bf16(gp, 512, gp, 256, dp, 516, 4, 256, st) == EALIGN
    torch.cuda.synchronize()
    assert h.untouched() and dgu.untouched()


# ---------------------------------------------------------------------------------------------------------------------
# CE loss
# ---------------------------------------------------------------------------------------------------------------------
def ce_inputs(rows, V, g, spread=True):
    lg = torch.randn(rows, V, device="cuda", generator=g) * 2
    if spread:
        lg[1::4] = lg[1::4] * 10 + 1e4                    # offset by 1e4 with a wide spread
    labels = torch.randint(0, V, (rows,), device="cuda", generator=g)
    labels[3::7] = -100
    if rows > 5:
        labels[5] = V + 5                                 # outside the vocabulary: ignored and not counted
    return lg, labels


def ce_ref(lg, labels):
    """fp64 loss rows, softmax, lse and the per-row bound dlse of the module docstring."""
    rows, V = lg.shape
    ld = lg.double()
    mx = ld.amax(-1, keepdim=True)
    e = torch.exp(ld - mx)
    S = e.sum(-1, keepdim=True)
    lse = mx + torch.log(S)
    p = e / S
    dlse = (-(-V // 512) + 21) * U + (p * (4 * U + U * (ld - mx).abs())).sum(-1, keepdim=True) \
        + 2 * U * torch.log(S).abs() + U * lse.abs()
    valid = (labels >= 0) & (labels < V)
    lab = labels.clamp(0, V - 1)
    loss_r = (lse[:, 0] - ld.gather(1, lab[:, None])[:, 0]) * valid
    return loss_r, p, lse, dlse, valid, lab


def ce_call(lg, labels, n_valid, loss_sum, dl):
    rows, V = lg.shape
    return _lib.lib().vllm_ce_loss_f32(lg.data_ptr(), lg.stride(0), labels.data_ptr(),
                                       None if n_valid is None else n_valid.data_ptr(), rows, V, loss_sum.data_ptr(),
                                       None if dl is None else dl.data_ptr(), 0 if dl is None else dl.stride(0), stream())


@pytest.mark.parametrize("V", [1, 511, 32026, 92544])
def test_ce_loss_vs_fp64(V):
    """The loss and dlogits against fp64 on pitched logits with NaN in the gap and pitched dlogits whose gap stays
    untouched; ignored rows (-100, and a label >= V) give exact 0 rows; `ops.ce_loss` and `CrossEntropyFn` divide by
    the same count."""
    from visionllm_b200 import ops
    from visionllm_b200.train import CrossEntropyFn
    g = gen(V)
    rows = 64
    lg, labels = ce_inputs(rows, V, g)
    _, lgv = pitched(lg, (V + 3) // 4 * 4 + 4)
    valid_n = int(((labels >= 0) & (labels < V)).sum())
    n_valid = torch.tensor([valid_n], device="cuda")
    loss_sum = torch.zeros(1, device="cuda")
    dl = Out(rows, V, (V + 7) // 8 * 8 + 8)
    assert ce_call(lgv, labels, n_valid, loss_sum, dl.view) == 0
    torch.cuda.synchronize()
    y = dl.check(f"dlogits V={V}")
    loss_r, p, lse, dlse, valid, lab = ce_ref(lg, labels)
    n = valid_n
    E_loss = ((dlse[:, 0] + U * loss_r.abs()) * valid).sum() + n * U * loss_r.abs().sum()
    within(loss_sum, loss_r.sum().reshape(1), E_loss.reshape(1), "ce_loss_sum", f"V={V}")
    onehot = torch.zeros_like(p).scatter_(1, lab[:, None], 1.0)
    z = (p - onehot) / n
    ld = lg.double()
    E = (1.25 * (p * (dlse + U * (ld - lse).abs() + 4 * U) + 3 * U * (p - onehot).abs()) + 2.0 ** -140) / n
    rounds(y[valid], z[valid], E[valid], "ce_dlogits", f"V={V}")
    assert (y[~valid] == 0).all(), "ignored rows are not exact 0"
    # the two wrappers: the same denominator, and their stated all-ignored results
    want = loss_r.sum() / n
    l_ops = ops.ce_loss(lgv, labels)
    l_fn = CrossEntropyFn.apply(lgv, labels)
    within(l_ops.reshape(1), want.reshape(1), (E_loss / n + U * want.abs()).reshape(1), "ce_loss_mean", f"V={V}")
    within(l_fn.reshape(1), want.reshape(1), (E_loss / n + U * want.abs()).reshape(1), "ce_loss_mean", f"V={V} train")
    none = torch.full_like(labels, -100)
    none[0] = V
    assert math.isnan(float(ops.ce_loss(lgv, none))), "ops.ce_loss over no valid row is not nan (torch's value)"
    x = lgv.detach().requires_grad_(True)
    l0 = CrossEntropyFn.apply(x, none)
    l0.backward()
    assert float(l0) == 0.0 and (x.grad == 0).all(), "CrossEntropyFn over no valid row is not 0 with a zero gradient"


@pytest.mark.parametrize("V", [32026, 92544])
def test_cross_entropy_upstream_gradient_in_fp32(V):
    """(loss * c).backward() scales dlogits by c in fp32: within two bf16 roundings of c (softmax - onehot) / n, with
    no bias (mean signed relative error <= 2^-12; a bf16 c would give 2^-9 at c = 1/3).  c = 1 leaves the kernel's
    dlogits as they are, bit for bit."""
    from visionllm_b200.train import CrossEntropyFn
    g = gen(V + 1)
    rows = 256
    lg, labels = ce_inputs(rows, V, g, spread=False)
    buf, lgv = pitched(lg, (V + 3) // 4 * 4)
    loss_r, p, lse, dlse, valid, lab = ce_ref(lg, labels)
    n = int(valid.sum())
    onehot = torch.zeros_like(p).scatter_(1, lab[:, None], 1.0)
    z1 = (p - onehot) / n
    E1 = (1.25 * (p * (dlse + U * (lg.double() - lse).abs() + 4 * U) + 3 * U * (p - onehot).abs()) + 2.0 ** -140) / n
    direct = Out(rows, V, (V + 7) // 8 * 8)
    assert ce_call(lgv, labels, torch.tensor([n], device="cuda"), torch.zeros(1, device="cuda"), direct.view) == 0
    for c in (1.0, 1 / 3, 0.1):
        x = lgv.detach().requires_grad_(True)
        (CrossEntropyFn.apply(x, labels) * c).backward()
        y = x.grad                                        # autograd casts the bf16 dlogits to the fp32 leaf's dtype
        if c == 1.0:
            assert same_bits(y.contiguous(), direct.view.float()), "dloss = 1 changed dlogits"
            continue
        y = y[valid].double()
        z, e1 = c * z1[valid], c * E1[valid]
        a1 = e1 + c * 0.5 * bf16_ulp(z1[valid].abs() + E1[valid])
        allow = (a1 + 0.5 * bf16_ulp(z.abs() + a1) + U * z.abs()) * (1 + 2.0 ** -20)
        err = (y - z).abs()
        note_ratio("ce_dloss_scale", float((err / allow).max()))
        assert bool((err <= allow).all()), f"c={c}: {int((err > allow).sum())} elements beyond two bf16 roundings"
        nz = z != 0
        bias = float(((y[nz] - z[nz]) / z[nz]).mean())
        assert abs(bias) <= 2.0 ** -12, f"c={c}: mean signed relative error {bias:.3g}"


# ---------------------------------------------------------------------------------------------------------------------
# RoPE backward and head stacking
# ---------------------------------------------------------------------------------------------------------------------
def hf_rope_grad(xq, cos, sin, heads, D, gy):
    """torch autograd of the HF bf16 formula on the first `heads` heads of the packed rows (the rest pass through)."""
    T = xq.shape[0]
    x = xq.detach().clone().requires_grad_(True)
    v = x[:, :heads * D].view(T, heads, D)
    rot = torch.cat((-v[..., D // 2:], v[..., :D // 2]), -1)
    out = torch.cat(((v * cos[:, None] + rot * sin[:, None]).reshape(T, -1), x[:, heads * D:]), 1)
    out.backward(gy)
    return out.detach(), x.grad


@pytest.mark.parametrize("nq,nkv", [(4, 4), (6, 2)])
@pytest.mark.parametrize("D", [64, 128])
def test_rope_backward_bit_identical_to_hf_autograd(D, nq, nkv):
    """RopeFn and QKVRopeFn (identity projection, so its dgrad GEMM returns the rotated gradient exactly) give the
    gradient of HF's bf16 formula bit for bit on the q and k heads; the v heads' gradient passes through."""
    from visionllm_b200 import train as TR
    from visionllm_b200.llama import rope_tables
    g = gen(D + nq)
    T = 300
    W = (nq + 2 * nkv) * D
    cos, sin = rope_tables(torch.arange(T, device="cuda") * 7 + 3, D, 10000.0, torch.bfloat16)
    neg_sin = (-sin).contiguous()
    xq = (torch.randn(T, W, device="cuda", generator=g) * 2).bfloat16()
    gy = (torch.randn(T, W, device="cuda", generator=g)).bfloat16()
    want_out, want = hf_rope_grad(xq, cos, sin, nq + nkv, D, gy)
    for have_neg in (False, True):
        x = xq.clone().requires_grad_(True)
        out = TR.RopeFn.apply(x, cos, sin, nq + nkv, D, neg_sin if have_neg else None)
        out.backward(gy)
        assert torch.equal(out.detach(), want_out), "RopeFn forward != HF formula"
        assert torch.equal(x.grad, want), f"RopeFn backward != HF autograd (neg_sin given: {have_neg})"
    eye = torch.eye(W, device="cuda", dtype=torch.bfloat16)
    x = xq.clone().requires_grad_(True)
    out = TR.QKVRopeFn.apply(x, eye, cos, sin, neg_sin, nq + nkv, D)
    out.backward(gy.clone())                              # rotated in place by the backward
    assert torch.equal(out.detach(), want_out), "QKVRopeFn forward != HF formula"
    assert torch.equal(x.grad, want), "QKVRopeFn backward != HF autograd"
    assert torch.equal(x.grad[:, (nq + nkv) * D:], gy[:, (nq + nkv) * D:]), "v heads' gradient changed"


@pytest.mark.parametrize("parts", [1, 3])
def test_head_stack_matches_permute_and_round_trips(parts):
    from visionllm_b200 import train as TR
    g = gen(parts)
    B, T, H, D = 2, 272, 5, 128
    x = torch.randn(B, T, parts, H, D, device="cuda", generator=g).bfloat16()
    st = TR.head_stack(x, B, T, parts, H, D, True)
    assert same_bits(st, x.permute(2, 0, 3, 1, 4).contiguous()), "stacked != permute"
    back = TR.head_stack(st, B, T, parts, H, D, False)
    assert same_bits(back, x), "round trip is not exact"
