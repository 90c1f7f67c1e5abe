"""GPU: the memory-bound row kernels of the forward path against float64 references of the same ops on the same bf16
inputs, with exact probes, bit-identities and sentinel checks of every byte around their outputs.

Kernels: RMSNorm, LayerNorm (+GELU, +residual, row gather), the pixel-shuffle LayerNorm, GroupNorm (+ReLU, padded
grids), the depthwise KxK conv, the FPN upsample-add, DCNv3 prep / blend, the TP reduce + RMSNorm and RoPE.

One checker, `rounds` (tests/bf16_rounding.py, shared with the training kernels' contract): a bf16 output y "rounds z
within E" (z the float64 reference, E a bound of the kernel's fp32 error before its final bf16 rounding) when
  (a) |y - z| <= E + ulp_bf16(|z| + E) / 2, and
  (b) y == RN_bf16(z) wherever no bf16 rounding midpoint lies in [z - E, z + E].
(b) is the sharp part: away from ties the output is the correctly rounded float64 value, bit for bit (values compared,
so +0 == -0).  RMSNorm and the upsample-add round twice; their inner bf16 value has at most two candidates, and the
outer operation (a bf16 x bf16 product, a bf16 + bf16 sum) is exact in fp32 and rounded once, so `rounds_twice`
accepts y = RN(outer(c)) for every candidate c the inner check allows and requires c = RN(z_inner) away from ties.

u = 2^-24.  d is the longest fp32 summation chain of a row reduction; in `launch_norm` (csrc/fused_ops.cu) it is
8 * VPT + 5 + TPR / 32 for the (VPT, TPR) the width selects, at most 77.  A re-tile must update `norm_chain`.  Bounds:
  RMSNorm     z_n = x * r, r = 1 / sqrt(mean(x^2) + eps); inner E_n = (d + 5) u |z_n|; then bf16(w * bf16(x r)).
  LayerNorm   z = (x - mu) r w + b;  E = |w| r (dmu + rho |x - mu|) + 4u (|(x - mu) r w| + |b|) with
              dmu = (d + 1) u mean|x| and rho = (d + 6) u + dmu^2 / (2 (var + eps)).
              GELU: 1.13 E + 4u |gelu(z)| + 2^-23 |z| (erff's absolute error where 1 + erf cancels).
              residual: E + u (|z| + |res|) around z + res.
  GroupNorm   the LayerNorm form with dmu = (t + 4) u mean|x| and rho = 2^-22 + (t + 4) u mean(x^2) / (var + eps): the
              statistics are one-pass fp32 (sum, sum of squares) per thread, so E[x^2] - mu^2 cancels by mean(x^2) / var.
              t = 8 * ceil(ceil(hw / chunks) / ppi) is the longest per-thread chain under the current chunking.
  dwconv      z = b + sum w x;  E = (K^2 + 2) u (|b| + sum |w x|).
  upsample    source index and lambda in fp32 exactly as ATen's CUDA kernel computes them (src = fma(scale, d + 0.5,
              -0.5)); taps combined in float64, inner E = 4u sum |lambda x|; then bf16(lateral + bf16(interp)).
  DCNv3 prep  offsets bit-exact; softmax within ((taps + 8) + |m_j - max| + max_k |m_k - max|) u z (the exponent's
              fp32 subtraction carries u |m - max| into exp); sigmoid within 8u z.
  DCNv3 blend E = 4u (|core (1 - s)| + |xproj s|); no scale: bit-exact bf16(core).
  TP reduce   x' rounds x + sum slots within (n_slots + 1) u (|x| + sum |slot|); every dst holds the RMSNorm contract
              of the observed x' (d = 8 VPT + 13), and all dsts are identical.
  RoPE        bit-exact against the HF bf16 formula on both kernels.

`pytest -s` prints, per family, the worst observed err / E (err = |y - z| - ulp_bf16(y) / 2, a lower bound of the
kernel's error before its last rounding) and the fraction of elements whose E interval held a rounding midpoint.  On an
NVIDIA H100 80GB HBM3 at 700 W the worst is 0.53 (LayerNorm + residual); GroupNorm's one-pass term makes about half of
its elements ties at hw = 65536.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from visionllm_b200 import _lib
from bf16_rounding import U, bf16_ulp, note_ratio, print_report, rn_bf16, rounds, rounds_mask, rounds_twice, rounds_twice_mask  # noqa: E501

gpu = pytest.mark.gpu
EINVAL, EUNSUPPORTED, EALIGN = -1, -2, -3
NAN = float("nan")
SENTINEL = 4320.0                  # exact in bf16; a non-zero border the upsample-add must leave alone


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("row kernels")


# ---- CPU cases for the checker itself ----
def _grid_values():
    z = torch.linspace(-3.0, 3.0, 20001, dtype=torch.float64) * 1.37 + 0.001
    return z[z != 0]


def test_checker_accepts_the_correct_rounding():
    z = _grid_values()
    ok, _ = rounds_mask(rn_bf16(z), z, 4 * U * z.abs())
    assert bool(ok.all())
    assert torch.equal(rn_bf16(torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(2.0 - 2.0 ** -9)],
                                            dtype=torch.float64)),
                       torch.tensor([1.0, 1.0 + 2 * 2.0 ** -7, -2.0], dtype=torch.float64))   # ties to even, binade carry


def test_checker_accepts_the_far_neighbour_only_near_a_midpoint():
    m = torch.tensor([1.0 + 2.0 ** -8, 3.0 + 2.0 ** -7, -0.75 - 2.0 ** -9], dtype=torch.float64)   # midpoints
    q = bf16_ulp(m)
    z = m + q * 2.0 ** -6                      # just above the midpoint: RN(z) is the upper neighbour
    far = m - q / 2                            # the lower neighbour
    assert not torch.equal(far, rn_bf16(z))
    ok_in, tie = rounds_mask(far, z, q * 2.0 ** -5)       # E reaches the midpoint
    assert bool(ok_in.all()) and bool(tie.all())
    ok_out, tie = rounds_mask(far, z, q * 2.0 ** -7)      # E stops short of it
    assert not bool(ok_out.any()) and not bool(tie.any())
    # the two-step form: the far inner candidate only at a tie
    outer = lambda c: rn_bf16(c * -2.0)                   # noqa: E731
    assert bool(rounds_twice_mask(outer(far), z, q * 2.0 ** -5, outer)[0].all())
    assert not bool(rounds_twice_mask(outer(far), z, q * 2.0 ** -7, outer)[0].any())


def test_checker_rejects_an_ulp_off():
    v = rn_bf16(_grid_values())
    z = v + 0.1 * bf16_ulp(v)                             # a tenth of an ulp off a bf16 value: far from every midpoint
    for y in (v + bf16_ulp(v), v - bf16_ulp(v)):
        ok, tie = rounds_mask(y, z, 64 * U * z.abs())
        assert not bool(ok.any()) and not bool(tie.any())
        ok, _ = rounds_twice_mask(rn_bf16(2 * y), z, 64 * U * z.abs(), lambda c: rn_bf16(2 * c))
        assert not bool(ok.any())
    ok, _ = rounds_mask(torch.full_like(z, NAN), z, 64 * U * z.abs())
    assert not bool(ok.any())


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
    """A [rows, cols] output view with row pitch ld, inside a NaN buffer with a NaN row above and below.  `check()`
    asserts every element of the view was written and nothing around it changed."""

    def __init__(self, rows, cols, ld=None, dtype=torch.bfloat16):
        ld = ld or cols
        self.buf = torch.full((rows + 2, ld), NAN, dtype=dtype, device="cuda")
        self.view = self.buf[1:rows + 1, :cols]
        self.before = bits(self.buf).clone()
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[1:rows + 1, :cols] = True

    def untouched(self):
        return torch.equal(bits(self.buf)[~self.inside], self.before[~self.inside]) and \
            torch.equal(bits(self.view), self.before[self.inside].view(self.view.shape))

    def check(self, what):
        assert not self.view.isnan().any(), f"{what}: {int(self.view.isnan().sum())} output elements never written"
        assert torch.equal(bits(self.buf)[~self.inside], self.before[~self.inside]), f"{what}: a store landed outside"
        return self.view


def vector(values):
    """A contiguous bf16 copy of `values` followed by NaN in memory: a read past its end poisons the result."""
    n = values.numel()
    buf = torch.full((n + 8,), NAN, dtype=torch.bfloat16, device="cuda")
    buf[:n] = values.flatten()
    return buf[:n]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def activations(kind, rows, cols, g):
    """normal N(0, 1); offset: mean 30 std; outlier: a few channels 300x the rest (the massive activations of ViT / LLM
    residual streams)."""
    x = torch.randn(rows, cols, device="cuda", generator=g)
    if kind == "offset":
        x = x + 30.0
    elif kind == "outlier":
        ch = torch.randperm(cols, device="cuda", generator=g)[:max(1, cols // 512)]
        x[:, ch] *= 300.0
    return x.bfloat16()


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm / LayerNorm (+GELU, +residual, gather)
# ---------------------------------------------------------------------------------------------------------------------
def norm_config(cols):
    """(VPT, TPR) that launch_norm picks for a row of `cols` columns."""
    nvec = cols // 8
    for lim, vpt, tpr in ((32, 1, 32), (64, 2, 32), (128, 4, 32), (256, 2, 128), (512, 4, 128), (1024, 8, 128)):
        if nvec <= lim:
            return vpt, tpr
    return 8, 256


def norm_chain(cols):
    vpt, tpr = norm_config(cols)
    return 8 * vpt + 5 + tpr // 32


def f32(v):
    return float(np.float32(v))


def check_rms(y, x, w, eps, d, family, what):
    xd = x.double()
    r = 1.0 / torch.sqrt((xd * xd).mean(-1, keepdim=True) + f32(eps))
    zn = xd * r
    wf = w.float()
    rounds_twice(y, zn, (d + 5) * U * zn.abs(), lambda c: (wf * c.float()).bfloat16().double(), family, what)


def ln_ref(x, w, b, eps, d):
    xd, wd, bd = x.double(), w.double(), b.double()
    mu = xd.mean(-1, keepdim=True)
    xc = xd - mu
    var = (xc * xc).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + f32(eps))
    a = xc * r * wd
    dmu = (d + 1) * U * xd.abs().mean(-1, keepdim=True)
    rho = (d + 6) * U + dmu * dmu / (2 * (var + f32(eps)))
    E = wd.abs() * r * (dmu + rho * xc.abs()) + 4 * U * (a.abs() + bd.abs())
    return a + bd, E


def gelu64(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def norm_call(kind, x, w, b, y, eps, res=None):
    L = _lib.lib()
    rows, cols = x.shape
    if kind == "rms":
        return L.vllm_rmsnorm_bf16(x.data_ptr(), x.stride(0), w.data_ptr(), y.data_ptr(), y.stride(0), rows, cols, eps,
                                   stream())
    if kind == "res":
        return L.vllm_layernorm_residual_bf16(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), res.data_ptr(),
                                              res.stride(0), y.data_ptr(), y.stride(0), rows, cols, eps, stream())
    fn = L.vllm_layernorm_gelu_bf16 if kind == "gelu" else L.vllm_layernorm_bf16
    return fn(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), y.data_ptr(), y.stride(0), rows, cols, eps, stream())


def check_norm(kind, y, x, w, b, eps, res, what):
    d = norm_chain(x.shape[1])
    if kind == "rms":
        return check_rms(y, x, w, eps, d, "rmsnorm", what)
    z, E = ln_ref(x, w, b, eps, d)
    if kind == "ln":
        rounds(y, z, E, "layernorm", what)
    elif kind == "gelu":
        rounds(y, gelu64(z), 1.13 * E + 4 * U * gelu64(z).abs() + 2.0 ** -23 * z.abs(), "layernorm_gelu", what)
    else:
        rd = res.double()
        rounds(y, z + rd, E + U * (z.abs() + rd.abs()), "layernorm_residual", what)


# both sides of every launch_norm boundary (cols / 8 = 1, 32 | 33, 64 | 65, 128 | 129, 256 | 257, 512 | 513,
# 1024 | 1025, 2048) and the product widths (CLIP / Swin / InternViT / Vicuna-7B/13B, InternLM2-20B, the 12800 bridge)
NORM_COLS = sorted({8 * n for n in (1, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024, 1025, 2048)}
                   | {256, 768, 1024, 1536, 3200, 4096, 5120, 6144, 12800})
NORM_KINDS = ["rms", "ln", "gelu", "res"]


@gpu
@pytest.mark.parametrize("cols", NORM_COLS)
@pytest.mark.parametrize("kind", NORM_KINDS)
def test_norm_rows_vs_fp64(kind, cols):
    """Every width config of launch_norm against fp64 on normal / offset / outlier rows, in pitched views with NaN in
    the input pitch gap, NaN after the weight and bias, and the output inside a NaN sentinel.  Zero rows (RMSNorm) and
    constant rows (LayerNorm) are exact.  Row slices, single rows, part-empty last CTAs (1 / 7 / 9 rows), contiguous
    views and in-place calls are bit-identical to the pitched call."""
    g = gen(cols * 7 + NORM_KINDS.index(kind))
    rows = 1025 if cols <= 4096 else 33
    ld = cols + 24
    eps = 1e-6 if kind in ("rms", "gelu") else 1e-5
    w = vector((1 + 0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16())
    b = vector((0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16())
    res = None
    if kind == "res":
        _, res = pitched(torch.randn(rows, cols, device="cuda", generator=g).bfloat16() * 2, ld + 8)
    for ik in ("normal", "offset", "outlier"):
        x = activations(ik, rows, cols, g)
        c = float(torch.tensor(1.5 + cols % 7 * 0.25).bfloat16())
        if kind == "rms":
            x[3] = 0                                     # exact zeros
        else:
            x[3] = c                                     # constant row: mu = c exactly, y = bf16(b) (+ res)
        _, xv = pitched(x, ld)
        out = Out(rows, cols, ld + 16)
        assert norm_call(kind, xv, w, b, out.view, eps, res) == 0
        torch.cuda.synchronize()
        y = out.check(f"{kind} {cols} {ik}")
        check_norm(kind, y, x, w, b, eps, res, f"cols={cols} {ik}")
        if kind == "rms":
            assert (y[3] == 0).all(), "RMSNorm of a zero row is not 0"
        elif kind == "ln":
            assert torch.equal(y[3], b), "LayerNorm of a constant row is not bias"
        elif kind == "res":
            assert torch.equal(y[3], (b.float() + res[3].float()).bfloat16()), "constant row: not bf16(b + res)"
        if ik != "normal":
            continue
        # bit-identities: slices / single rows / part-empty last CTAs, contiguous views, in place
        for lo, hi in ((0, 1), (2, 9), (rows - 7, rows), (rows - 9, rows), (5, 6)):
            o = Out(hi - lo, cols)
            assert norm_call(kind, xv[lo:hi], w, b, o.view, eps, None if res is None else res[lo:hi]) == 0
            assert same_bits(o.check("slice"), y[lo:hi]), f"rows {lo}:{hi} differ from the full call"
        xc = x.clone()
        o = Out(rows, cols)
        assert norm_call(kind, xc, w, b, o.view, eps, None if res is None else res.contiguous()) == 0
        assert same_bits(o.check("contiguous"), y), "contiguous views differ from pitched ones"
        buf, xi = pitched(x, ld)
        assert norm_call(kind, xi, w, b, xi, eps, res) == 0
        assert same_bits(xi, y), "in place differs from out of place"
        assert buf[:, cols:].isnan().all(), "the in-place call wrote into the pitch gap"
        if kind == "ln":                                 # the Swin window-partition gather: LN then gather, pads exact 0
            B, N = 2, min(rows // 2, 40)
            x3 = x[:B * N].reshape(B, N, cols).contiguous()
            idx = torch.cat([torch.randperm(N, device="cuda", generator=g), torch.tensor([N, N + 5, 10 ** 6], device="cuda")])
            from visionllm_b200 import ops
            got = ops.layernorm_gather(x3, idx, w, b, eps)
            want = torch.zeros_like(got)
            want[:, :N] = y[:B * N].reshape(B, N, cols)[:, idx[:N]]
            assert same_bits(got, want), "layernorm_gather != layernorm + gather"


@gpu
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("C", [8, 96, 256, 1024, 3200])
def test_pixel_shuffle_layernorm_vs_fp64(C, order):
    """The permutation exact, the LayerNorm(4C) under the LayerNorm bound (4C up to 12800; d = 8 VPT + 13 for the
    kernel's VPT and its 8-warp block sum)."""
    from visionllm_b200 import ops
    g = gen(C + order)
    tiles, gw, gh = 2, 8, 6
    skip = 1 if order == 0 else 0
    for ik in ("normal", "offset", "outlier"):
        hs = activations(ik, tiles * (skip + gw * gh), C, g).reshape(tiles, skip + gw * gh, C)
        x4 = hs[:, skip:].reshape(tiles, gw, gh, C)
        if order == 0:        # mv2.py pixel shuffle: row (a, b) = cat over (dy, dx) of token (2a + dy, 2b + dx)
            ref = torch.cat([x4[:, 0::2, 0::2], x4[:, 0::2, 1::2], x4[:, 1::2, 0::2], x4[:, 1::2, 1::2]], -1)
        else:                 # HF SwinPatchMerging
            ref = torch.cat([x4[:, 0::2, 0::2], x4[:, 1::2, 0::2], x4[:, 0::2, 1::2], x4[:, 1::2, 1::2]], -1)
        ref = ref.reshape(tiles, -1, 4 * C)
        assert torch.equal(ops.pixel_shuffle_rows(hs, skip, grid=(gw, gh), order=order), ref)
        w = vector((1 + 0.5 * torch.randn(4 * C, device="cuda", generator=g)).bfloat16())
        b = vector((0.5 * torch.randn(4 * C, device="cuda", generator=g)).bfloat16())
        y = ops.pixel_shuffle_rows(hs, skip, w, b, 1e-5, grid=(gw, gh), order=order)
        nvec = 4 * C // 8
        vpt = 2 if nvec <= 512 else (4 if nvec <= 1024 else 8)
        z, E = ln_ref(ref, w, b, 1e-5, 8 * vpt + 13)
        rounds(y, z, E, "pixel_shuffle_ln", f"C={C} order={order} {ik}")


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------
GN_HW = {1: (1, 1), 5: (1, 5), 777: (21, 37), 4096: (64, 64), 65536: (256, 256)}
GN_CASES = [(C, G, hw) for C, G in ((48, 1), (48, 6), (256, 1), (256, 32), (2048, 1), (2048, 32), (2048, 256))
            for hw in GN_HW if not (hw == 65536 and C == 2048)]


def gn_call(x, y, gamma, beta, n, h, w, w_pitch, img_pitch, C, G, eps, relu, ws, ws_bytes=None):
    return _lib.lib().vllm_groupnorm_nhwc_bf16_grid(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), n, h, w,
                                                   w_pitch, img_pitch, C, G, eps, relu, ws.data_ptr(),
                                                   ws.numel() if ws_bytes is None else ws_bytes, stream())


def gn_chain(hw, C):
    """Longest per-thread fp32 chain of gn_stats_kernel (csrc/groupnorm.cu chunking)."""
    c8 = C // 8
    ppi = 256 // c8
    chunks = min(max(-(-hw // (ppi * 8)), 1), 128)
    per = -(-hw // chunks)
    return 8 * -(-per // ppi)


def gn_inputs(kind, n, hw, C, G, g):
    if kind == "twolevel":                 # every group holds c and c + ulp(c): |mean| / std ~ 400
        c = torch.tensor([96.0, -200.0, 3.25], device="cuda")[torch.arange(G, device="cuda") % 3]
        c = c.repeat_interleave(C // G)
        hi = torch.rand(n, hw, C, device="cuda", generator=g) < 0.5
        return (c + hi * bf16_ulp(c.double()).float()).bfloat16()
    x = activations(kind, n * hw, C, g).reshape(n, hw, C)
    if kind == "offset":
        x = (x.float() + torch.randn(C, device="cuda", generator=g) * 5).bfloat16()   # per-group offsets differ
    return x


@gpu
@pytest.mark.parametrize("C,G,hw", GN_CASES)
def test_groupnorm_vs_fp64(C, G, hw):
    """Contiguous and padded-grid inputs (NaN outside the valid corner) against fp64, relu 0 / 1; a constant group gives
    exactly bf16(beta) (or its ReLU); padded == contiguous and two runs are bit-identical."""
    g = gen(C * 131 + G * 7 + hw)
    h, w = GN_HW[hw]
    n = 1 if hw == 65536 else 3
    cpg = C // G
    eps = 1e-5
    gamma = vector((1 + 0.5 * torch.randn(C, device="cuda", generator=g)).bfloat16())
    beta = vector((0.5 * torch.randn(C, device="cuda", generator=g)).bfloat16())
    ws = torch.empty(_lib.lib().vllm_groupnorm_workspace_bytes(n, G), dtype=torch.uint8, device="cuda")
    t = gn_chain(hw, C)
    for kind in ("normal", "offset", "outlier", "twolevel"):
        relu = int(kind in ("offset", "twolevel"))
        x = gn_inputs(kind, n, hw, C, G, g)
        if kind == "normal":
            x[0, :, :cpg] = 3.5                          # a constant group: mean exact, y = bf16(beta) exactly
        # padded grid: valid [h, w] corner of a [h + 2, w + 3] image, images 5 pixels apart beyond that
        wp, ip = w + 3, (h + 2) * (w + 3) + 5
        grid = torch.full((n, ip, C), NAN, dtype=torch.bfloat16, device="cuda")
        grid[:, :(h + 2) * wp].view(n, h + 2, wp, C)[:, :h, :w] = x.view(n, h, w, C)
        outs = []
        for src, wpi, ipi in ((x, w, hw), (grid, wp, ip)):
            o = Out(n * hw, C)
            assert gn_call(src, o.view, gamma, beta, n, h, w, wpi, ipi, C, G, eps, relu, ws) == 0
            outs.append(o.check(f"groupnorm {kind}").reshape(n, hw, C))
        y = outs[0]
        assert same_bits(outs[1], y), "padded grid != contiguous copy of its corner"
        o = Out(n * hw, C)
        assert gn_call(x, o.view, gamma, beta, n, h, w, w, hw, C, G, eps, relu, ws) == 0
        assert same_bits(o.check("rerun").reshape(n, hw, C), y), "two runs differ"
        # fp64 reference
        xd = x.double().reshape(n, hw, G, cpg)
        mu = xd.mean((1, 3), keepdim=True)
        xc = xd - mu
        var = (xc * xc).mean((1, 3), keepdim=True)
        r = 1.0 / torch.sqrt(var + f32(eps))
        gd, bd = gamma.double().reshape(G, cpg), beta.double().reshape(G, cpg)
        a = xc * r * gd
        dmu = (t + 4) * U * xd.abs().mean((1, 3), keepdim=True)
        rho = 2.0 ** -22 + (t + 4) * U * (xd * xd).mean((1, 3), keepdim=True) / (var + f32(eps))
        E = gd.abs() * r * (dmu + rho * xc.abs()) + 4 * U * (a.abs() + bd.abs())
        z = a + bd
        if relu:
            z = z.clamp(min=0)
        rounds(y.reshape(n, hw, G, cpg), z, E, "groupnorm", f"C={C} G={G} hw={hw} {kind} relu={relu}")
        if kind == "normal":
            want = beta[:cpg].expand(hw, cpg)
            assert torch.equal(y[0, :, :cpg], want), "constant group is not bf16(beta)"
    # the constant probe under ReLU
    x = gn_inputs("normal", n, hw, C, G, g)
    x[:, :, :cpg] = -0.75
    o = Out(n * hw, C)
    assert gn_call(x, o.view, gamma, beta, n, h, w, w, hw, C, G, eps, 1, ws) == 0
    y = o.check("relu probe").reshape(n, hw, C)
    assert torch.equal(y[:, :, :cpg], beta[:cpg].clamp(min=0).expand(n, hw, cpg))


# ---------------------------------------------------------------------------------------------------------------------
# depthwise conv
# ---------------------------------------------------------------------------------------------------------------------
def dw_call(x, wt, bias, y, K):
    B, H, W, C = x.shape
    return _lib.lib().vllm_dwconv_nhwc_bf16(x.data_ptr(), wt.data_ptr(), None if bias is None else bias.data_ptr(),
                                            y.data_ptr(), B, H, W, C, K, stream())


class FlatOut(Out):
    def __init__(self, shape, dtype=torch.bfloat16):
        n = math.prod(shape)
        super().__init__(1, n, dtype=dtype)
        self.view = self.buf[1, :n].view(shape)


@gpu
@pytest.mark.parametrize("C", [8, 24, 320])
@pytest.mark.parametrize("K", [3, 5, 7])
def test_dwconv_vs_fp64_and_impulses(K, C):
    """W in {1, 3, 4, 5, 9} (the TW = 4 pixel tile and its tails), H in {1, 2, 7} (maps smaller than K), bias or none,
    against fp64; then a single 1.0 pixel at the centre, a corner and an edge gives exactly bf16(bias + w[tap]) at every
    output it reaches and exactly bias elsewhere -- tap orientation and borders pinned."""
    g = gen(K * 1000 + C)
    R = K // 2
    wt = vector((torch.randn(K * K, C, device="cuda", generator=g) / K).bfloat16()).view(K * K, C)
    bias = vector((torch.randn(C, device="cuda", generator=g) * 0.5).bfloat16())
    w4 = wt.double().t().reshape(C, 1, K, K)
    for H in (1, 2, 7):
        for W in (1, 3, 4, 5, 9):
            x = activations("normal" if (H + W) % 2 else "outlier", 2 * H * W, C, g).reshape(2, H, W, C)
            for bb in (bias, None):
                o = FlatOut((2, H, W, C))
                assert dw_call(x, wt, bb, o.view, K) == 0
                y = o.check(f"dwconv K={K} {H}x{W}")
                xd = x.double().permute(0, 3, 1, 2)
                z = F.conv2d(xd, w4, None if bb is None else bb.double(), padding=R, groups=C).permute(0, 2, 3, 1)
                s = F.conv2d(xd.abs(), w4.abs(), None, padding=R, groups=C).permute(0, 2, 3, 1)
                if bb is not None:
                    s = s + bb.double().abs()
                rounds(y, z, (K * K + 2) * U * s, "dwconv", f"K={K} C={C} {H}x{W} bias={bb is not None}")
    H, W = 7, 9
    for ph, pw in ((3, 4), (0, 0), (6, 8), (0, 5), (4, 0)):
        x = torch.zeros(1, H, W, C, dtype=torch.bfloat16, device="cuda")
        x[0, ph, pw] = 1.0
        o = FlatOut((1, H, W, C))
        assert dw_call(x, wt, bias, o.view, K) == 0
        y = o.check("impulse")[0]
        want = bias.expand(H, W, C).clone()
        for h in range(H):
            for w in range(W):
                dy, dx = ph - h + R, pw - w + R
                if 0 <= dy < K and 0 <= dx < K:
                    want[h, w] = (bias.float() + wt[dy * K + dx].float()).bfloat16()
        assert torch.equal(y, want), f"impulse at ({ph}, {pw}): taps misplaced"


# ---------------------------------------------------------------------------------------------------------------------
# FPN upsample-add
# ---------------------------------------------------------------------------------------------------------------------
def up_axis(n_in, n_out):
    """ATen's upsample_bilinear2d source indices and weights (align_corners=False) in fp32, as the kernel computes them:
    scale = in / out, src = max(fma(scale, d + 0.5, -0.5), 0), i1 = i0 + (i0 < in - 1), lambda = src - i0."""
    s = np.float32(n_in) / np.float32(n_out)
    d = np.arange(n_out, dtype=np.float64)
    src = np.maximum((np.float64(s) * (d + 0.5) - 0.5).astype(np.float32), np.float32(0))   # one rounding: the FFMA
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    lam = (src - i0.astype(np.float32)).astype(np.float32)
    hl = (np.float32(1) - lam).astype(np.float32)
    t = lambda a: torch.from_numpy(a).cuda()                       # noqa: E731
    return t(i0), t(i1), t(lam.astype(np.float64)), t(hl.astype(np.float64))


def up_call(top, pitch, lat, out, B, Hi, Wi, Ho, Wo, C, pad):
    return _lib.lib().vllm_upsample_add_nhwc_bf16_ex(top.data_ptr(), pitch, lat.data_ptr(), out.data_ptr(), B, Hi, Wi, Ho,
                                                     Wo, C, pad, stream())


UP_CASES = [((8, 6), (16, 12)), ((5, 7), (13, 11)), ((16, 12), (5, 7)), ((1, 1), (4, 5)), ((3, 1), (7, 2))]


@gpu
@pytest.mark.parametrize("C", [8, 256])
@pytest.mark.parametrize("src,dst", UP_CASES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in UP_CASES])
def test_upsample_add_vs_fp64(src, dst, C):
    """x2, non-integer up and down ratios and a 1x1 source, top images `pitch` apart with NaN between them, out_pad 0
    and 2 (the border holds a non-zero sentinel that must stay); the padded interior equals the out_pad = 0 result; a
    constant top map gives exactly bf16(lateral + c)."""
    g = gen(C + src[0] * 31 + dst[1])
    (Hi, Wi), (Ho, Wo) = src, dst
    B = 2
    pitch = Hi * Wi * C + 24
    topbuf = torch.full((B, pitch), NAN, dtype=torch.bfloat16, device="cuda")
    topd = activations("outlier", B * Hi * Wi, C, g).reshape(B, Hi, Wi, C)
    topbuf[:, :Hi * Wi * C] = topd.reshape(B, -1)
    lat = (torch.randn(B, Ho, Wo, C, device="cuda", generator=g) * 3).bfloat16()
    o = FlatOut((B, Ho, Wo, C))
    assert up_call(topbuf, pitch, lat, o.view, B, Hi, Wi, Ho, Wo, C, 0) == 0
    y = o.check("upsample_add")
    y0, y1, ly, hy = up_axis(Hi, Ho)
    x0, x1, lx, hx = up_axis(Wi, Wo)
    T = topd.double()
    tap = lambda yi, xi: T[:, yi][:, :, xi]                     # noqa: E731
    hy_, ly_ = hy.view(1, -1, 1, 1), ly.view(1, -1, 1, 1)
    hx_, lx_ = hx.view(1, 1, -1, 1), lx.view(1, 1, -1, 1)
    a, b, c, d = tap(y0, x0), tap(y0, x1), tap(y1, x0), tap(y1, x1)
    z = hy_ * (hx_ * a + lx_ * b) + ly_ * (hx_ * c + lx_ * d)
    s = hy_ * (hx_ * a.abs() + lx_ * b.abs()) + ly_ * (hx_ * c.abs() + lx_ * d.abs())
    latf = lat.float()
    rounds_twice(y, z, 4 * U * s, lambda u: (latf + u.float()).bfloat16().double(), "upsample_add", f"{src}->{dst} C={C}")
    for pad in (2,):
        buf = torch.full((B, Ho + 2 * pad, Wo + 2 * pad, C), SENTINEL, dtype=torch.bfloat16, device="cuda")
        ob = FlatOut(buf.shape)
        ob.view.copy_(buf)
        ob.before = bits(ob.buf).clone()
        assert up_call(topbuf, pitch, lat, ob.view, B, Hi, Wi, Ho, Wo, C, pad) == 0
        torch.cuda.synchronize()
        assert torch.equal(bits(ob.buf)[~ob.inside], ob.before[~ob.inside]), "out_pad: a store landed outside the map"
        inner = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
        inner[:, pad:pad + Ho, pad:pad + Wo] = True
        assert (ob.view[~inner] == SENTINEL).all(), "out_pad: the border was written"
        assert same_bits(ob.view[:, pad:pad + Ho, pad:pad + Wo], y), "out_pad interior != out_pad 0"
    cst = torch.full((B, pitch), -2.375, dtype=torch.bfloat16, device="cuda")
    o = FlatOut((B, Ho, Wo, C))
    assert up_call(cst, pitch, lat, o.view, B, Hi, Wi, Ho, Wo, C, 0) == 0
    assert torch.equal(o.check("constant"), (latf - 2.375).bfloat16()), "constant map: not bf16(lateral + c)"


# ---------------------------------------------------------------------------------------------------------------------
# DCNv3 prep / blend
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("G,K,with_scale", [(10, 9, True), (2, 9, False), (4, 25, True), (7, 25, False)])
def test_dcnv3_prep_vs_fp64(G, K, with_scale):
    g = gen(G * K + with_scale)
    rows = 301
    need = G * K * 3 + (G if with_scale else 0)
    om = torch.randn(rows, need, device="cuda", generator=g) * 4
    L = _lib.lib()
    results = []
    for ld in (need, need + 13):                       # contiguous, and a pitch with NaN in the gap
        buf = torch.full((rows, ld), NAN, device="cuda")
        buf[:, :need] = om
        off, mask, sc = FlatOut((rows, G * K * 2), torch.float32), FlatOut((rows, G * K), torch.float32), \
            FlatOut((rows, G), torch.float32)
        assert L.vllm_dcnv3_prep_f32(buf.data_ptr(), ld, off.view.data_ptr(), mask.view.data_ptr(),
                                     sc.view.data_ptr() if with_scale else None, rows, G, K, stream()) == 0
        torch.cuda.synchronize()
        results.append((off.check("offset"), mask.check("mask"), sc.check("scale") if with_scale else None))
        if not with_scale:
            assert sc.untouched()
    (off, mask, sc), (off2, mask2, sc2) = results
    assert same_bits(off2, off) and same_bits(mask2, mask) and (sc is None or same_bits(sc2, sc)), "pitched != contiguous"
    assert same_bits(off, om[:, :G * K * 2]), "offsets are not a copy"
    m = om[:, G * K * 2:G * K * 3].double().reshape(rows, G, K)
    z = torch.softmax(m, -1)
    dm = m - m.amax(-1, keepdim=True)
    rel = (K + 8 + dm.abs() + dm.abs().amax(-1, keepdim=True)) * U
    err = (mask.double().reshape(rows, G, K) - z).abs() / (rel * z)
    note_ratio("dcnv3_prep_softmax", float(err.max()))
    assert float(err.max()) <= 1.0, f"softmax off by {float(err.max())} bounds"
    if with_scale:
        zs = torch.sigmoid(om[:, G * K * 3:].double())
        err = (sc.double() - zs).abs() / (8 * U * zs)
        note_ratio("dcnv3_prep_sigmoid", float(err.max()))
        assert float(err.max()) <= 1.0, f"sigmoid off by {float(err.max())} bounds"


@gpu
@pytest.mark.parametrize("C,gc", [(320, 32), (16, 16), (2560, 160), (24, 8)])
def test_dcnv3_blend_vs_fp64(C, gc):
    g = gen(C + gc)
    rows = 777
    G = C // gc
    core = torch.randn(rows, C, device="cuda", generator=g) * 3
    xp = torch.randn(rows, C, device="cuda", generator=g) * 3
    s = torch.sigmoid(torch.randn(rows, G, device="cuda", generator=g) * 3)
    sbuf = torch.full((rows * G + 8,), NAN, device="cuda")
    sbuf[:rows * G] = s.flatten()
    L = _lib.lib()
    o = FlatOut((rows, C))
    assert L.vllm_dcnv3_blend_bf16(core.data_ptr(), xp.data_ptr(), sbuf.data_ptr(), o.view.data_ptr(), rows, C, gc,
                                   stream()) == 0
    y = o.check("blend")
    sd = s.double().repeat_interleave(gc, -1)
    a, b = core.double() * (1 - sd), xp.double() * sd
    rounds(y, a + b, 4 * U * (a.abs() + b.abs()), "dcnv3_blend", f"C={C} gc={gc}")
    o = FlatOut((rows, C))
    assert L.vllm_dcnv3_blend_bf16(core.data_ptr(), None, None, o.view.data_ptr(), rows, C, gc, stream()) == 0
    assert same_bits(o.check("blend, no scale"), core.bfloat16()), "blend without scale != bf16(core)"


# ---------------------------------------------------------------------------------------------------------------------
# TP reduce + RMSNorm (local slots, one GPU)
# ---------------------------------------------------------------------------------------------------------------------
def tp_call(slots, n_slots, x, w, eps, dsts, ld_dst, rows, cols):
    arr = (ctypes.c_void_p * max(len(dsts), 1))(*[d.data_ptr() for d in dsts])
    return _lib.lib().vllm_tp_reduce_norm_bf16(None if slots is None else slots.data_ptr(), n_slots,
                                               0 if slots is None else slots.stride(0), x.data_ptr(), w.data_ptr(), eps,
                                               arr, len(dsts), ld_dst, None, 0, None, 0, rows, cols, stream())


@gpu
@pytest.mark.parametrize("cols", [256, 2048, 2056, 4096, 5120, 8192])
@pytest.mark.parametrize("n_slots", [0, 1, 3, 7])
def test_tp_reduce_norm_vs_fp64(n_slots, cols):
    g = gen(cols + n_slots)
    rows = 1025 if cols <= 2048 else 130
    eps = 1e-5
    x = activations("outlier", rows, cols, g)
    x0 = x.clone()
    slots = (torch.randn(max(n_slots, 1), rows, cols, device="cuda", generator=g) * 2).bfloat16()
    w = vector((1 + 0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16())
    ld = cols + 8
    outs = [Out(rows, cols, ld) for _ in range(2)]
    assert tp_call(slots if n_slots else None, n_slots, x, w, eps, [o.view for o in outs], ld, rows, cols) == 0
    torch.cuda.synchronize()
    ys = [o.check(f"tp dst {i}") for i, o in enumerate(outs)]
    assert same_bits(ys[1], ys[0]), "the destinations differ"
    if n_slots == 0:
        assert same_bits(x, x0), "no slots: x must stay untouched"
    else:
        sd = slots[:n_slots].double()
        z = x0.double() + sd.sum(0)
        rounds(x, z, (n_slots + 1) * U * (x0.double().abs() + sd.abs().sum(0)), "tp_reduce", f"slots={n_slots} cols={cols}")
    nvec = cols // 8
    vpt = 1 if nvec <= 256 else (2 if nvec <= 512 else 4)
    check_rms(ys[0], x, w, eps, 8 * vpt + 13, "tp_norm", f"slots={n_slots} cols={cols}")
    one = Out(rows, cols, ld)                           # one destination: the same rows
    x1 = x0.clone()
    assert tp_call(slots if n_slots else None, n_slots, x1, w, eps, [one.view], ld, rows, cols) == 0
    assert same_bits(one.check("tp one dst"), ys[0]) and same_bits(x1, x)


# ---------------------------------------------------------------------------------------------------------------------
# RoPE
# ---------------------------------------------------------------------------------------------------------------------
def rope_call(x, ld, cos, sin, tokens, heads, D):
    return _lib.lib().vllm_rope_bf16(x.data_ptr(), ld, cos.data_ptr(), sin.data_ptr(), tokens, heads, D, stream())


@gpu
@pytest.mark.parametrize("D", [20, 64, 128, 256])
def test_rope_both_kernels_bit_exact(D):
    """q and k slices of a packed qkv row against the HF bf16 formula, bit for bit: rope_vec_kernel (16-byte rows) and
    rope_kernel (D % 16 != 0, a pitch that is not a multiple of 8, or a base 2 elements off 16 bytes) on copies of the
    same data.  The v slice and the pitch gap stay untouched."""
    g = gen(D)
    T, H = 77, 3
    HD = H * D
    inv = 1.0 / (10000 ** (torch.arange(0, D, 2, device="cuda").double() / D))
    fr = torch.outer(torch.arange(T, device="cuda").double() * 37 + 5, inv)
    emb = torch.cat((fr, fr), -1)
    cos, sin = vector(emb.cos().bfloat16().flatten()).view(T, D), vector(emb.sin().bfloat16().flatten()).view(T, D)
    qkv = (torch.randn(T, 3 * HD, device="cuda", generator=g) * 4).bfloat16()

    def hf(q):
        qh = q.view(T, H, D)
        rot = torch.cat((-qh[..., D // 2:], qh[..., :D // 2]), -1)
        return ((qh * cos[:, None]) + (rot * sin[:, None])).view(T, HD)

    want = torch.cat([hf(qkv[:, :HD].contiguous()), hf(qkv[:, HD:2 * HD].contiguous()), qkv[:, 2 * HD:]], 1)
    ld8 = (3 * HD + 7) // 8 * 8 + 8
    # (row start in elements, row pitch): 16-byte rows (the vector kernel when D % 16 == 0), a pitch that is not a
    # multiple of 8, a base 2 elements (4 bytes) off 16-byte alignment -- the last two always run the scalar kernel
    for base, ld in ((0, ld8), (0, ld8 + 2), (2, ld8)):
        buf = torch.full(((T + 1) * (ld + base),), NAN, dtype=torch.bfloat16, device="cuda")
        rowsv = buf[base:base + T * ld].view(T, ld)
        rowsv[:, :3 * HD] = qkv
        before = bits(buf).clone()
        assert rope_call(rowsv[:, :HD], ld, cos, sin, T, H, D) == 0             # q
        assert rope_call(rowsv[:, HD:2 * HD], ld, cos, sin, T, H, D) == 0       # k
        torch.cuda.synchronize()
        assert same_bits(rowsv[:, :3 * HD], want), f"RoPE D={D} base={base} ld={ld} != HF formula"
        keep = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
        keep[base:base + T * ld].view(T, ld)[:, :2 * HD] = False
        assert torch.equal(bits(buf)[keep], before[keep]), "RoPE wrote outside q / k"
    # one token at a time == the full call
    for t in (0, 40, T - 1):
        xt = qkv[t:t + 1, :HD].clone()
        assert rope_call(xt, HD, cos[t:t + 1], sin[t:t + 1], 1, H, D) == 0
        assert same_bits(xt, want[t:t + 1, :HD])


# ---------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_rejections_leave_the_output_untouched():
    L = _lib.lib()
    st = stream()
    x = torch.randn(16, 16400, device="cuda").bfloat16()
    w = torch.ones(16400, device="cuda").bfloat16()
    o = Out(4, 16400)
    y = o.view
    xp, wp, yp = x.data_ptr(), w.data_ptr(), y.data_ptr()
    lx, ly = x.stride(0), y.stride(0)
    norm_cases = {
        "cols > 16384": (xp, lx, yp, ly, 16392, EUNSUPPORTED),
        "cols % 8": (xp, lx, yp, ly, 100, EUNSUPPORTED),
        "x misaligned": (xp + 2, lx, yp, ly, 256, EALIGN),
        "y misaligned": (xp, lx, yp + 2, ly, 256, EALIGN),
        "ldx % 8": (xp, 260, yp, ly, 256, EALIGN),
        "ldy % 8": (xp, lx, yp, 260, 256, EALIGN),
    }
    for what, (a, la, c, lc, cols, rc) in norm_cases.items():
        assert L.vllm_rmsnorm_bf16(a, la, wp, c, lc, 4, cols, 1e-6, st) == rc, f"rmsnorm {what}"
        assert L.vllm_layernorm_bf16(a, la, wp, wp, c, lc, 4, cols, 1e-6, st) == rc, f"layernorm {what}"
        assert L.vllm_layernorm_gelu_bf16(a, la, wp, wp, c, lc, 4, cols, 1e-6, st) == rc, f"layernorm_gelu {what}"
        assert L.vllm_layernorm_residual_bf16(a, la, wp, wp, xp, lx, c, lc, 4, cols, 1e-6, st) == rc, f"ln_res {what}"
    assert L.vllm_rmsnorm_bf16(xp, lx, wp + 2, yp, ly, 4, 256, 1e-6, st) == EINVAL
    assert L.vllm_layernorm_bf16(xp, lx, wp, wp + 2, yp, ly, 4, 256, 1e-6, st) == EINVAL
    assert L.vllm_layernorm_residual_bf16(xp, lx, wp, wp, xp + 2, lx, yp, ly, 4, 256, 1e-6, st) == EALIGN
    assert L.vllm_layernorm_residual_bf16(xp, lx, wp, wp, xp, 260, yp, ly, 4, 256, 1e-6, st) == EALIGN
    # TP reduce-norm: cols > 8192, ld_dst % 8, misaligned x
    arr = (ctypes.c_void_p * 1)(yp)
    assert L.vllm_tp_reduce_norm_bf16(None, 0, 0, xp, wp, 1e-5, arr, 1, ly, None, 0, None, 0, 4, 8200, st) == EUNSUPPORTED
    assert L.vllm_tp_reduce_norm_bf16(None, 0, 0, xp, wp, 1e-5, arr, 1, 260, None, 0, None, 0, 4, 256, st) == EUNSUPPORTED
    assert L.vllm_tp_reduce_norm_bf16(None, 0, 0, xp + 2, wp, 1e-5, arr, 1, ly, None, 0, None, 0, 4, 256, st) == EALIGN
    # GroupNorm: cpg % 8, C > 2048, groups > 256, short workspace, misaligned
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    gn = lambda C, G, wsb=ws.numel(), xx=xp, yy=yp: L.vllm_groupnorm_nhwc_bf16_grid(   # noqa: E731
        xx, yy, wp, wp, 1, 2, 2, 2, 4, C, G, 1e-5, 0, ws.data_ptr(), wsb, st)
    assert gn(48, 12) == EUNSUPPORTED
    assert gn(2056, 1) == EUNSUPPORTED
    assert gn(4096, 512) == EUNSUPPORTED
    assert gn(2048, 512) == EUNSUPPORTED
    assert gn(256, 32, wsb=8 * 32 - 1) == EINVAL
    assert gn(256, 32, xx=xp + 2) == EALIGN
    assert gn(256, 32, yy=yp + 2) == EALIGN
    # depthwise conv: K not in {3, 5, 7}; upsample-add: C % 8
    for K in (1, 4, 9):
        assert L.vllm_dwconv_nhwc_bf16(xp, wp, None, yp, 1, 4, 4, 16, K, st) == EUNSUPPORTED
    assert L.vllm_dwconv_nhwc_bf16(xp, wp, None, yp, 1, 4, 4, 12, 3, st) == EUNSUPPORTED
    assert L.vllm_upsample_add_nhwc_bf16_ex(xp, 4 * 12, xp, yp, 1, 2, 2, 4, 4, 12, 0, st) == EUNSUPPORTED
    assert L.vllm_upsample_add_nhwc_bf16_ex(xp + 2, 4 * 16, xp, yp, 1, 2, 2, 4, 4, 16, 0, st) == EALIGN
    assert L.vllm_rope_bf16(yp, 64, wp, wp, 4, 1, 18, st) == EUNSUPPORTED
    torch.cuda.synchronize()
    assert o.untouched(), "a rejected call wrote to its output"
