"""GPU: every deformable-sampling kernel -- MSDA forward (fp32 warp gather, bf16-value warp gather, TMA / cp.async window
kernel, fused module-input kernel, strict fp32 / fp64), MSDA backward (fp32, fp64), DCNv3 forward (fast, strict) and
backward -- against a float64 reference of the same operation on the same inputs, with exact probes, bit-identities and
NaN sentinels around every output.

The reference does the geometry in the kernels' own fp32 sequence (h_im = fl(fl(loc_y H) - 0.5) as separate torch ops,
the range test, floor, lh = h_im - h_low, the corner bits; DCNv3's p0 - ((dil (k - 1)) >> 1) s + (i dil + off) s with
every step rounded) and asserts that it equals `ms_deform_attn_sample_indices` element for element; everything after
the geometry is float64: hh = 1 - lh, the corner weights, t = a w_corner v, z = sum t, A = sum |t|.

Bounds (u = 2^-24, g(n) = n u / (1 - n u); no max|ref| term):
  forward      E = g(d + c) A.  c = 4: the roundings of 1 - lh, 1 - lw, hh hw and (hh hw) a that every term carries
               (strict kernels: c = 5, their w v product is rounded too).  d is the longest fp32 chain a term passes
               through: K FMAs + 2 shuffle adds (fp32 warp and window kernels, DCNv3 fast), ceil(K / 2) FMAs + 3 shuffle
               adds (bf16 value: each lane sums every second sample), K adds + 3 corner adds (strict).  fp64 entry
               points: the same with u = 2^-53.  A bf16 output must round z within E (`rounds` of bf16_rounding.py):
               away from a rounding midpoint it is RN_bf16(z) bit for bit.
  backward     grad_value: g(hits + 5) sum |w g a| per element (hits = corner terms landing on it; tg a, the three
               weight roundings and w tga; the atomics add in any order).  grad_attn_weight: g(ceil(D / 32) + 5 + 8)
               sum_c |g_c| sum_corner |w v| (5: the butterfly; 8: the weight, w v, three corner adds, g ...).
               grad_sampling_loc: the same form over W |a| sum_c |g_c| sum_corner |other-axis weight v| (H for y;
               DCNv3: |offset_scale| |mask|).
  fused QP     the glue's softmax / offset normalisation are bit-identical to the torch ops (checked here through the
               returned weights), so z is built from the glue's loc / attw and the bf16-value bound applies.

`pytest -s` prints the worst err / E per family; DESIGN.md section 4 lists the values measured on an H100.
"""
import math

import pytest
import torch

from visionllm_b200 import _lib
from bf16_rounding import U, print_report, rn_bf16, rounds, within

pytestmark = pytest.mark.gpu
EINVAL, EUNSUPPORTED, EALIGN = -1, -2, -3
NAN = float("nan")
DEV = "cuda"
U64 = 2.0 ** -53
CORNERS = ((0, 0, 2), (0, 1, 4), (1, 0, 8), (1, 1, 16))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("deformable-sampling kernels")


def g_(n, u=U):
    return n * u / (1 - n * u)


def stream():
    return torch.cuda.current_stream().cuda_stream


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a.contiguous()), bits(b.contiguous()))


class Out:
    """An output of `shape` inside a buffer with `pad` NaN elements before and after it, prefilled with `fill`.
    `check()` asserts that every element was written (no NaN left) and that nothing around it changed."""

    def __init__(self, shape, dtype=torch.float32, fill=NAN, pad=64):
        self.n, self.pad = math.prod(shape), pad
        self.buf = torch.full((self.n + 2 * pad,), NAN, dtype=dtype, device=DEV)
        self.buf[pad:pad + self.n] = fill
        self.view = self.buf[pad:pad + self.n].view(shape)
        self.before = bits(self.buf).clone()

    def untouched(self):
        return torch.equal(bits(self.buf), self.before)

    def check(self, what):
        torch.cuda.synchronize()
        b, p, n = bits(self.buf), self.pad, self.n
        assert torch.equal(b[:p], self.before[:p]) and torch.equal(b[p + n:], self.before[p + n:]), \
            f"{what}: a store landed outside the output"
        assert not self.view.isnan().any(), f"{what}: {int(self.view.isnan().sum())} output elements never written"
        return self.view


# ---------------------------------------------------------------------------------------------------------------------
# MSDA: inputs, entry points, reference
# ---------------------------------------------------------------------------------------------------------------------
class Pyr:
    def __init__(self, shapes_l):
        self.list = [tuple(s) for s in shapes_l]
        self.L = len(shapes_l)
        self.host = torch.tensor(self.list, dtype=torch.int64)
        self.dev = self.host.to(DEV)
        self.lsi = torch.cat((self.dev.new_zeros(1), self.dev.prod(1).cumsum(0)[:-1])).contiguous()
        self.S = int(self.host.prod(1).sum())


PYR = {
    "pow2": [(16, 16), (8, 8), (4, 4), (2, 2)],
    "npot": [(25, 34), (13, 17), (7, 9), (4, 5)],
    "gdino": [(100, 167), (50, 84), (25, 42), (13, 21)],           # 800 x 1333 image
    "thin": [(1, 7), (9, 1), (3, 3), (1, 1)],                       # levels with H = 1 or W = 1
}


def pixel_centres(pyr):
    refs = []
    for (H, W) in pyr.list:
        ys, xs = torch.meshgrid(torch.arange(H, device=DEV, dtype=torch.float32),
                                torch.arange(W, device=DEV, dtype=torch.float32), indexing="ij")
        refs.append(torch.stack(((xs + 0.5) / W, (ys + 0.5) / H), -1).reshape(-1, 2))
    return torch.cat(refs, 0)


def msda_inputs(pyr, N, M, Lq, P, seed, D=32, sigma=0.03):
    """value exact in bf16 (every path reads the same numbers), scaled by 2^k per (pixel, head) so that outputs span
    many magnitudes; encoder-like locations (pixel centres + noise, 3 % anywhere) when Lq == S, else uniform over
    [-0.15, 1.15); attention weights with a 2^k spread per (query, head)."""
    g = gen(seed)
    L = pyr.L
    value = torch.randn(N, pyr.S, M, D, device=DEV, generator=g)
    value = value * torch.exp2(torch.randint(-6, 7, (N, pyr.S, M, 1), device=DEV, generator=g).float())
    value = value.bfloat16().float()
    if Lq == pyr.S:
        ref = pixel_centres(pyr)[None, :, None, None, None, :]
        loc = ref + torch.randn(N, Lq, M, L, P, 2, device=DEV, generator=g) * sigma
        wild = torch.rand(N, Lq, M, L, P, 1, device=DEV, generator=g) < 0.03
        loc = torch.where(wild, torch.rand(N, Lq, M, L, P, 2, device=DEV, generator=g) * 1.4 - 0.2, loc)
    else:
        loc = torch.rand(N, Lq, M, L, P, 2, device=DEV, generator=g) * 1.3 - 0.15
    attw = torch.softmax(torch.randn(N, Lq, M, L * P, device=DEV, generator=g), -1)
    attw = attw * torch.exp2(torch.randint(-6, 3, (N, Lq, M, 1), device=DEV, generator=g).float())
    return value.contiguous(), loc.contiguous(), attw.view(N, Lq, M, L, P).contiguous()


def dims(value, loc):
    N, S, M, D = value.shape
    return N, S, M, D, loc.shape[3], loc.shape[1], loc.shape[4]


def f32_fwd(value, pyr, loc, attw, variant=_lib.MSDA_DEFAULT, flags=0, hint=True, vptr=None):
    N, S, M, D, L, Lq, P = dims(value, loc)
    o = Out((N, Lq, M * D))
    with _lib.knob("msda_set_variant", variant):
        rc = _lib.lib().vllm_msda_forward_f32(vptr or value.data_ptr(), pyr.dev.data_ptr(), pyr.lsi.data_ptr(),
                                              loc.data_ptr(), attw.data_ptr(), o.view.data_ptr(), N, S, M, D, L, Lq, P,
                                              pyr.host.data_ptr() if hint else None, flags, stream())
    assert rc == 0, rc
    return o.check(f"msda f32 variant={variant} flags={flags} hint={hint}")


def f64_fwd(value, pyr, loc, attw):
    N, S, M, D, L, Lq, P = dims(value, loc)
    o = Out((N, Lq, M * D), torch.float64)
    v, lo, a = value.double(), loc.double(), attw.double()
    assert _lib.lib().vllm_msda_forward_f64(v.data_ptr(), pyr.dev.data_ptr(), pyr.lsi.data_ptr(), lo.data_ptr(),
                                            a.data_ptr(), o.view.data_ptr(), N, S, M, D, L, Lq, P, stream()) == 0
    return o.check("msda f64")


def bf16_fwd(value, pyr, loc, attw, out_bf16, window=True, hint=True):
    N, S, M, D, L, Lq, P = dims(value, loc)
    v = value.bfloat16()
    o = Out((N, Lq, M * D), torch.bfloat16 if out_bf16 else torch.float32)
    with _lib.knob("msda_set_variant", _lib.MSDA_DEFAULT if window else _lib.MSDA_BF16_NO_WINDOW):
        rc = _lib.lib().vllm_msda_forward_bf16v(v.data_ptr(), pyr.dev.data_ptr(), pyr.lsi.data_ptr(), loc.data_ptr(),
                                                attw.data_ptr(), o.view.data_ptr(), int(out_bf16), N, S, M, D, L, Lq, P,
                                                pyr.host.data_ptr() if hint else None, stream())
    assert rc == 0, rc
    return o.check(f"msda bf16v out_bf16={out_bf16} window={window}")


def msda_geom(loc, pyr):
    """(h_low, w_low, mask, lh, lw) [N, Lq, M, L, P] by the kernels' sequence in loc's dtype; h_low = w_low = 0 and
    lh = lw = 0 outside the range (what the index dump writes)."""
    dt, dev = loc.dtype, loc.device
    H = torch.tensor([h for h, _ in pyr.list], dtype=dt, device=dev)[:, None]
    W = torch.tensor([w for _, w in pyr.list], dtype=dt, device=dev)[:, None]
    h_im = torch.sub(torch.mul(loc[..., 1], H), 0.5)
    w_im = torch.sub(torch.mul(loc[..., 0], W), 0.5)
    inr = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
    hf, wf = torch.floor(h_im.float()), torch.floor(w_im.float())          # floorf((float)h_im), as the kernels
    zero = torch.zeros((), dtype=dt, device=dev)
    lh = torch.where(inr, torch.sub(h_im, hf.to(dt)), zero)
    lw = torch.where(inr, torch.sub(w_im, wf.to(dt)), zero)
    hl = torch.where(inr, torch.nan_to_num(hf).long(), 0)
    wl = torch.where(inr, torch.nan_to_num(wf).long(), 0)
    Hi, Wi = H.long(), W.long()
    m = inr.int()
    m |= (inr & (hl >= 0) & (wl >= 0)).int() << 1
    m |= (inr & (hl >= 0) & (wl + 1 <= Wi - 1)).int() << 2
    m |= (inr & (hl + 1 <= Hi - 1) & (wl >= 0)).int() << 3
    m |= (inr & (hl + 1 <= Hi - 1) & (wl + 1 <= Wi - 1)).int() << 4
    return hl, wl, m, lh, lw


def check_geom_is_the_devices(loc, pyr, geom):
    import visionllm_b200.msda as ext
    dump = ext.ms_deform_attn_sample_indices(pyr.dev, loc).long()
    hl, wl, m = geom[:3]
    assert torch.equal(dump[..., 0], hl) and torch.equal(dump[..., 1], wl) and torch.equal(dump[..., 2], m.long()), \
        "the reference geometry differs from the kernels' msda_geom"


def corner_terms(lh, lw):
    """Per corner: (weight, d weight / d lw, d weight / d lh) in float64."""
    lh, lw = lh.double(), lw.double()
    hh, hw = 1 - lh, 1 - lw
    return ((hh * hw, -hh, -hw), (hh * lw, hh, -lw), (lh * hw, -lh, hw), (lh * lw, lh, lw))


def msda_rows(pyr, N, M, geom):
    """Flat row index (b, pixel, head) of the low corner of every sample, and the level widths."""
    hl, wl = geom[:2]
    dev = hl.device
    Wl = torch.tensor([w for _, w in pyr.list], device=dev)[:, None]
    start = pyr.lsi.to(dev)[:, None]
    b = torch.arange(N, device=dev).view(N, 1, 1, 1, 1)
    m = torch.arange(M, device=dev).view(1, 1, M, 1, 1)
    return (b * pyr.S + start + hl * Wl + wl) * M + m, Wl


def msda_ref(value, pyr, loc, attw, geom=None):
    """(z, A) [N, Lq, M * D] float64 of the forward."""
    N, S, M, D, L, Lq, P = dims(value, loc)
    geom = geom if geom is not None else msda_geom(loc, pyr)
    mk = geom[2]
    base, Wl = msda_rows(pyr, N, M, geom)
    v = value.double().reshape(-1, D)
    a = attw.double()
    z = torch.zeros(N, Lq, M, D, dtype=torch.float64, device=value.device)
    A = torch.zeros_like(z)
    for (dh, dw, bit), (w, _, _) in zip(CORNERS, corner_terms(*geom[3:])):
        ok = (mk & bit) != 0
        idx = torch.where(ok, base + (dh * Wl + dw) * M, 0).reshape(-1)
        t = torch.where(ok, w * a, 0.0).view(N, Lq, M, L * P, 1)
        prod = torch.where(ok.view(N, Lq, M, L * P, 1), t * v[idx].view(N, Lq, M, L * P, D), 0.0)
        z += prod.sum(3)
        A += prod.abs().sum(3)
        del prod
    return z.view(N, Lq, M * D), A.view(N, Lq, M * D)


def fwd_E(kind, K, A):
    d, c, u = {"f32": (K + 2, 4, U), "bf16": (-(-K // 2) + 3, 4, U), "strict": (K + 3, 5, U),
               "f64": (K + 3, 5, U64)}[kind]
    return g_(d + c, u) * A


# ---------------------------------------------------------------------------------------------------------------------
# MSDA forward vs fp64, every entry point
# ---------------------------------------------------------------------------------------------------------------------
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_many(M, Lq=900):
    """The smallest batch at which Lq queries no longer count as "few" (csrc/msda.cu: ceil(Lq/128) M N < 4 SMs)."""
    return -(-4 * sms() // (-(-Lq // 128) * M))


FWD_CASES = {   # pyramid, N, M, Lq (None: the encoder shape Lq == S), P
    "k1": ([(16, 16)], 2, 8, None, 1),
    "k2_dec": ([(16, 16), (8, 8)], 3, 1, 37, 1),
    "k3": (PYR["npot"][:3], 1, 8, None, 1),
    "k5_l5": ([(12, 20), (6, 10), (3, 5), (2, 3), (1, 2)], 2, 8, None, 1),    # L = 5: no window kernel
    "k5_l1": ([(25, 34)], 1, 1, None, 5),
    "k16_pow2": (PYR["pow2"], 2, 8, None, 4),
    "k16_npot": (PYR["npot"], 2, 8, None, 4),
    "k16_thin_enc": (PYR["thin"], 2, 8, None, 4),
    "k16_thin_dec": (PYR["thin"], 2, 1, 50, 4),
    "k31": ([(17, 23)], 1, 1, None, 31),
    "k32": ([(13, 17), (7, 9)], 2, 8, None, 16),
    "k33": (PYR["npot"][:3], 2, 8, 20, 11),                                   # K > 32: strict fallback
    "gdino_dec_few": (PYR["gdino"], 2, 8, 900, 4),
    "gdino_dec_many": (PYR["gdino"], "many", 8, 900, 4),
}


@pytest.mark.parametrize("case", list(FWD_CASES))
def test_msda_forward_vs_fp64(case):
    """Every forward entry point against the fp64 reference (fp32 warp kernel with and without the hint, the fp32 window
    kernel, bf16 value with fp32 / bf16 out with and without the window kernel, strict fp32 and fp64), each output
    NaN-prefilled inside a sentinel.  Bit-identities: the fp32 fast paths agree, window == global for bf16 values,
    bf16 out == the same kernel's fp32 out rounded to nearest, bf16 value == fp32 at K = 1."""
    shapes_l, N, M, Lq, P = FWD_CASES[case]
    pyr = Pyr(shapes_l)
    N = n_many(M) if N == "many" else N
    Lq = pyr.S if Lq is None else Lq
    K = pyr.L * P
    value, loc, attw = msda_inputs(pyr, N, M, Lq, P, seed=len(case) * 31 + K)
    geom = msda_geom(loc, pyr)
    check_geom_is_the_devices(loc, pyr, geom)
    z, A = msda_ref(value, pyr, loc, attw, geom)
    within(f32_fwd(value, pyr, loc, attw, flags=1), z, fwd_E("strict", K, A), "msda_fwd_strict_f32", case)
    z64, A64 = msda_ref(value, pyr, loc.double(), attw.double())
    within(f64_fwd(value, pyr, loc, attw), z64, fwd_E("f64", K, A64), "msda_fwd_f64", case)
    fast = f32_fwd(value, pyr, loc, attw)
    if K > 32:
        assert same_bits(fast, f32_fwd(value, pyr, loc, attw, flags=1)), "K > 32 does not take the strict kernel"
        return
    within(fast, z, fwd_E("f32", K, A), "msda_fwd_f32", case)
    assert same_bits(fast, f32_fwd(value, pyr, loc, attw, _lib.MSDA_NO_HINT)), f"{case}: hint changed the result"
    assert same_bits(fast, f32_fwd(value, pyr, loc, attw, hint=False)), f"{case}: NULL hint changed the result"
    assert same_bits(fast, f32_fwd(value, pyr, loc, attw, _lib.MSDA_FP32_WINDOW)), f"{case}: fp32 window != warp"
    for window in (True, False):
        y32 = bf16_fwd(value, pyr, loc, attw, False, window)
        y16 = bf16_fwd(value, pyr, loc, attw, True, window)
        within(y32, z, fwd_E("bf16", K, A), "msda_fwd_bf16v", f"{case} window={window}")
        rounds(y16, z, fwd_E("bf16", K, A), "msda_fwd_bf16v_bf16out", f"{case} window={window}")
        assert same_bits(y16, y32.bfloat16()), f"{case}: bf16 out != fp32 out rounded (window={window})"
        if window:
            w32, w16 = y32, y16
        else:
            assert same_bits(w32, y32) and same_bits(w16, y16), f"{case}: window kernel != global path"
    assert same_bits(bf16_fwd(value, pyr, loc, attw, False, hint=False), w32), f"{case}: NULL hint != hint (bf16v)"
    if K == 1:
        assert same_bits(w32, fast), "bf16 value != fp32 value at K = 1"


def test_region_encoder_shape_with_padded_samples():
    """The region encoder's grid_sample pooling: one level, 16 points, trailing samples padded with weight 0 (their
    locations anywhere, NaN included)."""
    pyr = Pyr([(24, 24)])
    N, M, Lq, P = 3, 8, 100, 16
    value, loc, attw = msda_inputs(pyr, N, M, Lq, P, seed=5)
    attw[..., 12:] = 0.0
    loc[:, ::3, :, :, 12:] = NAN
    geom = msda_geom(loc, pyr)
    z, A = msda_ref(value, pyr, loc, attw, geom)
    for variant in (_lib.MSDA_DEFAULT, _lib.MSDA_NO_HINT):
        within(f32_fwd(value, pyr, loc, attw, variant), z, fwd_E("f32", P, A), "msda_fwd_f32", "region encoder")
    within(f32_fwd(value, pyr, loc, attw, flags=1), z, fwd_E("strict", P, A), "msda_fwd_strict_f32", "region encoder")
    rounds(bf16_fwd(value, pyr, loc, attw, True), z, fwd_E("bf16", P, A), "msda_fwd_bf16v_bf16out", "region encoder")


def test_full_encoder_shape():
    """N = 2, S = 21760, M = 8: coverage and NaN sentinels on every query, fp64 on a seeded subset of 4096 queries,
    window == global path bit for bit (fp32 and bf16 values)."""
    pyr = Pyr([(128, 128), (64, 64), (32, 32), (16, 16)])
    N, M, P = 2, 8, 4
    value, loc, attw = msda_inputs(pyr, N, M, pyr.S, P, seed=77, sigma=0.02)
    q = torch.randperm(pyr.S, device=DEV, generator=gen(3))[:4096].sort().values
    ls, aws = loc[:, q].contiguous(), attw[:, q].contiguous()
    geom = msda_geom(ls, pyr)
    check_geom_is_the_devices(ls, pyr, geom)
    z, A = msda_ref(value, pyr, ls, aws, geom)
    fast = f32_fwd(value, pyr, loc, attw)
    within(fast[:, q], z, fwd_E("f32", 16, A), "msda_fwd_f32", "encoder")
    assert same_bits(fast, f32_fwd(value, pyr, loc, attw, _lib.MSDA_FP32_WINDOW)), "fp32 window != warp (encoder)"
    assert same_bits(fast, f32_fwd(value, pyr, loc, attw, hint=False)), "NULL hint != hint (encoder)"
    within(f32_fwd(value, pyr, loc, attw, flags=1)[:, q], z, fwd_E("strict", 16, A), "msda_fwd_strict_f32", "encoder")
    y32, y16 = bf16_fwd(value, pyr, loc, attw, False), bf16_fwd(value, pyr, loc, attw, True)
    within(y32[:, q], z, fwd_E("bf16", 16, A), "msda_fwd_bf16v", "encoder")
    rounds(y16[:, q], z, fwd_E("bf16", 16, A), "msda_fwd_bf16v_bf16out", "encoder")
    assert same_bits(y16, y32.bfloat16())
    assert same_bits(y32, bf16_fwd(value, pyr, loc, attw, False, window=False)), "bf16 window != global (encoder)"


WINDOWS = [(0, 0, 0), (2, 3, 1), (4, 4, 2), (8, 16, 1), (16, 16, 12)]


def test_window_fill_masks_and_geometries_are_bit_identical_to_the_global_path():
    """Every fill mask 0..15 of vllm_msda_set_window_fill and window geometries small enough that many samples fall
    outside their window (the in-kernel global re-base) give the global path's bits, fp32 and bf16 values."""
    pyr = Pyr(PYR["npot"])
    value, loc, attw = msda_inputs(pyr, 2, 8, pyr.S, 4, seed=9, sigma=0.05)
    base32 = f32_fwd(value, pyr, loc, attw, _lib.MSDA_NO_HINT)
    base16 = bf16_fwd(value, pyr, loc, attw, False, window=False)
    base16b = bf16_fwd(value, pyr, loc, attw, True, window=False)
    for window in WINDOWS:
        for fill in range(16):
            with _lib.knob("msda_set_window", *window), _lib.knob("msda_set_window_fill", fill):
                what = f"window={window} fill={fill}"
                assert same_bits(f32_fwd(value, pyr, loc, attw, _lib.MSDA_FP32_WINDOW), base32), "fp32 " + what
                assert same_bits(bf16_fwd(value, pyr, loc, attw, False), base16), "bf16 value " + what
                if fill in (0, 5, 15):
                    assert same_bits(bf16_fwd(value, pyr, loc, attw, True), base16b), "bf16 out " + what


# ---------------------------------------------------------------------------------------------------------------------
# exact probes
# ---------------------------------------------------------------------------------------------------------------------
def fingerprint(pyr, N, M, D=32):
    """value[b, pixel, m, c]: small integers (exact in bf16) that name the batch entry, level, row, column and head,
    one field per channel, a mix of all of them on the others."""
    rows = []
    for l, (H, W) in enumerate(pyr.list):
        h, w = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
        rows.append(torch.stack((torch.full_like(h, l), h, w), -1).reshape(-1, 3))
    lhw = torch.cat(rows, 0)[None, :, None, None, :]                              # [1, S, 1, 1, 3]
    b = torch.arange(N, device=DEV).view(N, 1, 1, 1)
    m = torch.arange(M, device=DEV).view(1, 1, M, 1)
    c = torch.arange(D, device=DEV).view(1, 1, 1, D)
    l, h, w = lhw[..., 0], lhw[..., 1], lhw[..., 2]
    mix = (b * 13 + l * 7 + h * 3 + w * 5 + m * 11 + c) % 251 + 1
    field = torch.stack(torch.broadcast_tensors(b + 1, l + 1, h + 1, w + 1, m + 1, mix, mix, mix), 0)
    v = field.gather(0, (c % 8).expand(1, *field.shape[1:]))[0]
    return v.float().contiguous()


def coord_for(target, n):
    """fp32 x with fl(fl(x n) - 0.5) == target (element-wise), searched over 64 ulps either side of (target + 0.5) / n;
    NaN where none exists."""
    t = target.float()
    nf = torch.full_like(t, float(n)) if not torch.is_tensor(n) else n.float().expand_as(t)
    x0 = ((t.double() + 0.5) / nf.double()).float()
    found = torch.full_like(t, NAN)
    up, dn = x0.clone(), x0.clone()
    hit = lambda x: torch.sub(torch.mul(x, nf), 0.5) == t                       # noqa: E731
    found = torch.where(hit(x0), x0, found)
    for _ in range(64):
        up, dn = torch.nextafter(up, torch.full_like(up, math.inf)), torch.nextafter(dn, torch.full_like(dn, -math.inf))
        found = torch.where(found.isnan() & hit(up), up, found)
        found = torch.where(found.isnan() & hit(dn), dn, found)
    return found


def border_targets(n):
    """h_im / w_im positions along an axis of n pixels: -1 (excluded), -1 + ulp, -0.5, 0, n - 1, n - 1/2, n - ulp, n
    (excluded)."""
    n32 = torch.tensor(float(n), device=DEV)
    return torch.stack((torch.tensor(-1.0, device=DEV), torch.nextafter(torch.tensor(-1.0, device=DEV), n32),
                        torch.tensor(-0.5, device=DEV), torch.tensor(0.0, device=DEV), n32 - 1, n32 - 0.5,
                        torch.nextafter(n32, torch.tensor(0.0, device=DEV)), n32))


def probe_inputs(pyr, N, M, P, seed):
    """One query per probe: sample (level l, point q % P) at an exact (h_im, w_im) target with a power-of-two weight
    (pixel centres, half pixels, every border position against a centre or half pixel on the other axis); every
    other sample out of range with a NaN weight.  Returns loc, attw, and the fraction of targets found."""
    g = gen(seed)
    targets = []                                                                   # (level, h_im, w_im)
    for l, (H, W) in enumerate(pyr.list):
        hb, wb = border_targets(H), border_targets(W)
        hc = torch.randint(0, H, (hb.numel(),), device=DEV, generator=g).float()
        wc = torch.randint(0, W, (wb.numel(),), device=DEV, generator=g).float()
        hs, ws = torch.arange(H, device=DEV).float(), torch.arange(W, device=DEV).float()
        hh, ww = torch.meshgrid(hs, ws, indexing="ij")
        for th, tw in ((hb, wc), (hc, wb), (hb, torch.full_like(hb, W / 2 - 0.5)),
                       (hh.flatten(), ww.flatten()), (hh.flatten() + 0.5, ww.flatten() + 0.5)):
            n = th.numel()
            targets.append(torch.stack((torch.full((n,), float(l), device=DEV), th, tw), -1))
    t = torch.cat(targets, 0)
    Lq = t.shape[0]
    lvl = t[:, 0].long()
    Hs = torch.tensor([h for h, _ in pyr.list], device=DEV)[lvl]
    Ws = torch.tensor([w for _, w in pyr.list], device=DEV)[lvl]
    y, x = coord_for(t[:, 1], Hs), coord_for(t[:, 2], Ws)
    ok = ~(y.isnan() | x.isnan())
    L = pyr.L
    loc = torch.full((Lq, L, P, 2), -7.0, device=DEV)                           # out of range on every level
    attw = torch.full((Lq, L, P), NAN, device=DEV)
    q = torch.arange(Lq, device=DEV)
    p = q % P
    loc[q, lvl, p, 0] = torch.where(ok, x, -7.0)
    loc[q, lvl, p, 1] = torch.where(ok, y, -7.0)
    attw[q, lvl, p] = torch.where(ok, torch.exp2(-(q % 4).float()), NAN)
    loc = loc[None, :, None].expand(N, Lq, M, L, P, 2).contiguous()
    attw = attw[None, :, None].expand(N, Lq, M, L, P).contiguous()
    return loc, attw, float(ok.float().mean())


@pytest.mark.parametrize("pyr_name", ["pow2", "npot", "thin"])
@pytest.mark.parametrize("M", [1, 8])
def test_msda_pixel_fingerprint_and_border_probes(pyr_name, M):
    """Fingerprint values, one sample per query at a pixel centre (lh = lw = 0 in fp32), a half pixel, or a border
    position, with a power-of-two weight: every path returns the exact value, i.e. the fingerprint of the intended
    pixel(s) -- a corner read from the neighbouring row, level, head or image shows.  The other samples lie out of range
    with NaN weights, which never reach the output."""
    pyr = Pyr(PYR[pyr_name])
    P = 4
    N = 2
    loc, attw, found = probe_inputs(pyr, N, M, P, seed=M)
    assert found > 0.9, f"only {found:.2f} of the probe positions exist in fp32"
    value = fingerprint(pyr, N, M)
    geom = msda_geom(loc, pyr)
    check_geom_is_the_devices(loc, pyr, geom)
    z, _ = msda_ref(value, pyr, loc, attw, geom)
    assert not z.isnan().any()
    what = f"{pyr_name} M={M}"
    for name, y in (("f32", f32_fwd(value, pyr, loc, attw)), ("nohint", f32_fwd(value, pyr, loc, attw, hint=False)),
                    ("window", f32_fwd(value, pyr, loc, attw, _lib.MSDA_FP32_WINDOW)),
                    ("strict", f32_fwd(value, pyr, loc, attw, flags=1)),
                    ("bf16v", bf16_fwd(value, pyr, loc, attw, False)),
                    ("bf16v_global", bf16_fwd(value, pyr, loc, attw, False, window=False))):
        assert torch.equal(y.double(), z), f"{name} {what}: {int((y.double() != z).sum())} probe outputs not exact"
    for window in (True, False):
        y = bf16_fwd(value, pyr, loc, attw, True, window)
        assert torch.equal(y.double(), rn_bf16(z)), f"bf16 out {what} window={window}: not RN_bf16 of the exact value"


# ---------------------------------------------------------------------------------------------------------------------
# MSDA bit-identities across batch, alignment, batch > 65535
# ---------------------------------------------------------------------------------------------------------------------
def test_msda_image_of_a_batch_equals_the_image_alone():
    """The batch size flips the few-queries rule and the tile shapes; per-pair arithmetic must not change."""
    pyr = Pyr(PYR["npot"])
    M = 8
    N = n_many(M, 200)
    value, loc, attw = msda_inputs(pyr, N, M, 200, 4, seed=41)
    enc_v, enc_l, enc_a = msda_inputs(pyr, 3, M, pyr.S, 4, seed=42)
    for v, lo, a in ((value, loc, attw), (enc_v, enc_l, enc_a)):
        full = {"f32": f32_fwd(v, pyr, lo, a), "bf16v": bf16_fwd(v, pyr, lo, a, False),
                "bf16v_bf16": bf16_fwd(v, pyr, lo, a, True)}
        for b in (0, v.shape[0] - 1):
            one = (v[b:b + 1].contiguous(), lo[b:b + 1].contiguous(), a[b:b + 1].contiguous())
            alone = {"f32": f32_fwd(*one[:1], pyr, *one[1:]), "bf16v": bf16_fwd(one[0], pyr, *one[1:], False),
                     "bf16v_bf16": bf16_fwd(one[0], pyr, *one[1:], True)}
            for k in full:
                assert same_bits(full[k][b:b + 1], alone[k]), f"{k}: image {b} of {v.shape[0]} != the image alone"


def test_msda_misaligned_value_takes_the_strict_kernel():
    pyr = Pyr(PYR["npot"][:2])
    value, loc, attw = msda_inputs(pyr, 2, 8, 40, 4, seed=8)
    buf = torch.empty(value.numel() + 1, device=DEV)
    buf[1:] = value.flatten()
    strict = f32_fwd(value, pyr, loc, attw, flags=1)
    assert same_bits(f32_fwd(value, pyr, loc, attw, vptr=buf[1:].data_ptr()), strict)


def test_msda_batch_over_65535():
    """N = 65536 at a 2 x 2 level: the grid's y extent is split into chunks, results are those of each image alone."""
    pyr = Pyr([(2, 2)])
    N, M, P = 65536, 1, 4
    value, loc, attw = msda_inputs(pyr, N, M, pyr.S, P, seed=65536)
    z, A = msda_ref(value, pyr, loc, attw)
    y = f32_fwd(value, pyr, loc, attw)
    within(y, z, fwd_E("f32", P, A), "msda_fwd_f32", "N = 65536")
    y16 = bf16_fwd(value, pyr, loc, attw, True)
    rounds(y16, z, fwd_E("bf16", P, A), "msda_fwd_bf16v_bf16out", "N = 65536")
    for b in (0, 65534, 65535):
        one = (value[b:b + 1].contiguous(), loc[b:b + 1].contiguous(), attw[b:b + 1].contiguous())
        assert same_bits(y[b:b + 1], f32_fwd(one[0], pyr, *one[1:])), f"f32 image {b}"
        assert same_bits(y16[b:b + 1], bf16_fwd(one[0], pyr, *one[1:], True)), f"bf16v image {b}"


# ---------------------------------------------------------------------------------------------------------------------
# fused module-input kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pyr_name", ["pow2", "npot"])
def test_fused_qp_kernel_vs_fp64(pyr_name):
    """Softmax / offset normalisation / reference add of the torch glue inside the window kernel: the returned weights
    are the glue's bits, the output is bf16v's on the glue's loc / attw (fp32 and bf16 out) and within the bf16v bound."""
    pyr = Pyr(PYR[pyr_name])
    N, M, L, P = 2, 8, 4, 4
    S = pyr.S
    g = gen(17)
    value = (torch.randn(N, S, M, 32, device=DEV, generator=g)).bfloat16()
    ld = M * 16 * 3 + 8
    qp = torch.full((N, S, ld), NAN, device=DEV).bfloat16()
    qp[..., :M * 32] = (torch.randn(N, S, M * 32, device=DEV, generator=g) * 2).bfloat16()
    qp[..., M * 32:M * 48] = (torch.randn(N, S, M * 16, device=DEV, generator=g) * 3).bfloat16()
    refp = (pixel_centres(pyr)[None, :, None, :].repeat(N, 1, L, 1) * 0.9).contiguous()
    # the glue (visionllm_b200/gdino.py, unfused branch)
    off = qp[..., :M * 32].reshape(N, S, M, L, P, 2)
    attw_g = torch.softmax(qp[..., M * 32:M * 48].reshape(N, S, M, L * P), -1).view(N, S, M, L, P)
    normalizer = torch.stack([pyr.dev[..., 1], pyr.dev[..., 0]], -1)
    loc = (refp[:, :, None, :, None, :] + off / normalizer[None, None, None, :, None, :]).float().contiguous()
    aw = attw_g.float().contiguous()
    z, A = msda_ref(value.float(), pyr, loc, aw)
    for out_bf16 in (False, True):
        o = Out((N, S, M * 32), torch.bfloat16 if out_bf16 else torch.float32)
        wo = Out((N, S, M, L, P), torch.bfloat16)
        assert _lib.lib().vllm_msda_forward_fused_bf16(
            value.data_ptr(), pyr.lsi.data_ptr(), qp.data_ptr(), ld, refp.data_ptr(), o.view.data_ptr(), int(out_bf16),
            wo.view.data_ptr(), N, S, M, 32, L, S, P, pyr.host.data_ptr(), stream()) == 0
        y, w = o.check("fused out"), wo.check("fused weights")
        assert same_bits(w, attw_g), "fused softmax != torch.softmax of the bf16 logits"
        assert same_bits(y, bf16_fwd(value.float(), pyr, loc, aw, out_bf16)), f"fused != bf16v on the glue (bf16 out {out_bf16})"
        if out_bf16:
            rounds(y, z, fwd_E("bf16", 16, A), "msda_fwd_fused_bf16out", pyr_name)
        else:
            within(y, z, fwd_E("bf16", 16, A), "msda_fwd_fused", pyr_name)


# ---------------------------------------------------------------------------------------------------------------------
# MSDA backward
# ---------------------------------------------------------------------------------------------------------------------
def msda_bwd(value, pyr, loc, attw, go, dt):
    N, S, M, D, L, Lq, P = dims(value, loc)
    v, lo, a, gr = (t.to(dt).contiguous() for t in (value, loc, attw, go))
    gv, gl, ga = Out(v.shape, dt, fill=0.0), Out(lo.shape, dt), Out(a.shape, dt)
    fn = _lib.lib().vllm_msda_backward_f32 if dt == torch.float32 else _lib.lib().vllm_msda_backward_f64
    assert fn(v.data_ptr(), pyr.dev.data_ptr(), pyr.lsi.data_ptr(), lo.data_ptr(), a.data_ptr(), gr.data_ptr(),
              gv.view.data_ptr(), gl.view.data_ptr(), ga.view.data_ptr(), N, S, M, D, L, Lq, P, stream()) == 0
    return gv.check("grad_value"), gl.check("grad_sampling_loc"), ga.check("grad_attn_weight")


def msda_bwd_ref(value, pyr, loc, attw, go):
    """z and sum-|term| of grad_value (+ hits per row), grad_sampling_loc (x, y) and grad_attn_weight, float64."""
    N, S, M, D, L, Lq, P = dims(value, loc)
    K = L * P
    geom = msda_geom(loc, pyr)
    mk = geom[2]
    base, Wl = msda_rows(pyr, N, M, geom)
    Hl = torch.tensor([h for h, _ in pyr.list], device=value.device)[:, None].double()
    v = value.double().reshape(-1, D)
    a = attw.double()
    gr = go.double().view(N, Lq, M, 1, D)
    gv = torch.zeros_like(v)
    gvA, hits = torch.zeros_like(v), torch.zeros(v.shape[0], dtype=torch.float64, device=v.device)
    zs = {k: torch.zeros(N, Lq, M, L, P, dtype=torch.float64, device=v.device) for k in ("a", "x", "y", "Aa", "Ax", "Ay")}
    for (dh, dw, bit), (w, cx, cy) in zip(CORNERS, corner_terms(*geom[3:])):
        ok = (mk & bit) != 0
        idx = torch.where(ok, base + (dh * Wl + dw) * M, 0)
        rows = torch.where(ok.view(N, Lq, M, K, 1), v[idx.reshape(-1)].view(N, Lq, M, K, D), 0.0)
        vg = (rows * gr).sum(-1).view(N, Lq, M, L, P)
        vgA = (rows.abs() * gr.abs()).sum(-1).view(N, Lq, M, L, P)
        zs["a"] += torch.where(ok, w * vg, 0.0)
        zs["Aa"] += torch.where(ok, (w * vgA).abs(), 0.0)
        zs["x"] += torch.where(ok, Wl * a * cx * vg, 0.0)
        zs["Ax"] += torch.where(ok, (Wl * a * cx).abs() * vgA, 0.0)
        zs["y"] += torch.where(ok, Hl * a * cy * vg, 0.0)
        zs["Ay"] += torch.where(ok, (Hl * a * cy).abs() * vgA, 0.0)
        sel = ok.reshape(-1)
        t = (torch.where(ok, w * a, 0.0).view(N, Lq, M, K, 1) * gr).reshape(-1, D)[sel]
        gv.index_add_(0, idx.reshape(-1)[sel], t)
        gvA.index_add_(0, idx.reshape(-1)[sel], t.abs())
        hits.index_add_(0, idx.reshape(-1)[sel], torch.ones(int(sel.sum()), dtype=torch.float64, device=v.device))
    gl = torch.stack((zs["x"], zs["y"]), -1)
    glA = torch.stack((zs["Ax"], zs["Ay"]), -1)
    return gv.view(value.shape), gvA.view(value.shape), hits.view(N, S, M, 1), gl, glA, zs["a"], zs["Aa"]


def check_bwd(got, ref, D, u, tag, what):
    gv, gl, ga = got
    zgv, Agv, hits, zgl, Agl, zga, Aga = ref
    within(gv, zgv, g_(hits + 5, u) * Agv, f"msda_bwd_grad_value_{tag}", what)
    c = -(-D // 32) + 5 + 8
    within(gl, zgl, g_(c, u) * Agl, f"msda_bwd_grad_loc_{tag}", what)
    within(ga, zga, g_(c, u) * Aga, f"msda_bwd_grad_attw_{tag}", what)


def bwd_inputs(pyr, N, M, Lq, P, D, seed):
    """Uniform locations, a third of all samples on one point (many atomics on the same pixels), and samples at every
    border position of every level."""
    value, loc, attw = msda_inputs(pyr, N, M, Lq, P, seed, D=D)
    loc[:, ::3] = torch.tensor([0.37, 0.61], device=DEV)
    for l, (H, W) in enumerate(pyr.list):
        bh, bw = border_targets(H)[1:-1], border_targets(W)[1:-1]
        n = min(bh.numel(), Lq)
        y, x = coord_for(bh[:n], H), coord_for(bw[:n], W)
        loc[:, 1:n + 1, :, l, 0, 0] = torch.where(x.isnan(), 0.5, x)[None, :, None]
        loc[:, 1:n + 1, :, l, 0, 1] = torch.where(y.isnan(), 0.5, y)[None, :, None]
    go = torch.randn(N, Lq, M * D, device=DEV, generator=gen(seed + 1))
    go = go * torch.exp2(torch.randint(-4, 5, (N, Lq, M, 1), device=DEV, generator=gen(seed + 2)).float()).repeat_interleave(D, -1).view(N, Lq, M * D)
    return value, loc.contiguous(), attw, go.contiguous()


@pytest.mark.parametrize("D", [4, 32, 71])
def test_msda_backward_vs_fp64(D):
    pyr = Pyr([(6, 5), (3, 4), (2, 2), (1, 1)])
    N, M, Lq, P = 2, 4, 60, 3
    value, loc, attw, go = bwd_inputs(pyr, N, M, Lq, P, D, seed=D)
    ref = msda_bwd_ref(value, pyr, loc, attw, go)
    got = msda_bwd(value, pyr, loc, attw, go, torch.float32)
    check_bwd(got, ref, D, U, "f32", f"D={D}")
    again = msda_bwd(value, pyr, loc, attw, go, torch.float32)
    assert same_bits(got[1], again[1]) and same_bits(got[2], again[2]), "grad_loc / grad_attw not reproducible"
    ref64 = msda_bwd_ref(value, pyr, loc.double(), attw.double(), go)
    check_bwd(msda_bwd(value, pyr, loc, attw, go, torch.float64), ref64, D, U64, "f64", f"D={D}")


def test_msda_backward_exact_probes():
    """One in-range sample at a half pixel (corner weights 1/4), a = 1/2, integer values and grad_out: every gradient is
    exact; out-of-range samples with NaN weights give exact zeros and leak nothing.  Power-of-two levels with H != W,
    so that the locations are exact in fp64 too and a grad_sampling_loc scaled by the wrong side shows."""
    pyr = Pyr([(8, 4), (2, 4)])
    N, M, Lq, P, D = 2, 2, 3, 2, 32
    value = torch.randint(-8, 9, (N, pyr.S, M, D), device=DEV, generator=gen(1)).float()
    loc = torch.full((N, Lq, M, 2, P, 2), -7.0, device=DEV)
    attw = torch.full((N, Lq, M, 2, P), NAN, device=DEV)
    for q, (l, hy, wx) in enumerate(((0, 2.5, 1.5), (1, 0.5, 2.5), (0, 4.5, 2.5))):
        H, W = pyr.list[l]
        xy = torch.cat((coord_for(torch.tensor([wx], device=DEV), W), coord_for(torch.tensor([hy], device=DEV), H)))
        assert not xy.isnan().any()
        loc[:, q, :, l, q % P] = xy
        attw[:, q, :, l, q % P] = 0.5
    go = torch.randint(-4, 5, (N, Lq, M * D), device=DEV, generator=gen(2)).float()
    zgv, _, _, zgl, _, zga, _ = msda_bwd_ref(value, pyr, loc, attw, go)
    for dt in (torch.float32, torch.float64):
        gv, gl, ga = msda_bwd(value, pyr, loc, attw, go, dt)
        assert torch.equal(gv.double(), zgv), f"grad_value not exact ({dt})"
        assert torch.equal(gl.double(), zgl), f"grad_sampling_loc not exact ({dt})"
        assert torch.equal(ga.double(), zga), f"grad_attn_weight not exact ({dt})"


# ---------------------------------------------------------------------------------------------------------------------
# DCNv3
# ---------------------------------------------------------------------------------------------------------------------
DCN_CASES = {   # N, H, W, G, C, kh, kw, sh, sw, ph, pw, dh, dw, offset_scale, offset amplitude
    "3x5": (2, 13, 19, 3, 32, 3, 5, 2, 1, 0, 2, 1, 2, 0.75, 3.0),
    "5x3": (1, 17, 11, 2, 32, 5, 3, 1, 2, 2, 0, 2, 1, 1.5, 4.0),
    "1x1": (2, 9, 7, 2, 32, 1, 1, 1, 1, 0, 0, 1, 1, 1.0, 2.0),
    "3x3": (1, 12, 12, 2, 32, 3, 3, 1, 1, 1, 1, 1, 1, 1.25, 3.0),
    "5x5": (1, 14, 10, 1, 32, 5, 5, 1, 1, 2, 2, 1, 1, 0.5, 2.0),
    "4x8": (1, 11, 13, 2, 32, 4, 8, 1, 1, 1, 3, 1, 1, 1.0, 2.0),           # K = 32
    "3x11": (1, 11, 13, 2, 32, 3, 11, 1, 1, 1, 5, 1, 1, 1.0, 2.0),         # K = 33: strict fallback
    "gc16": (2, 8, 9, 3, 16, 3, 5, 2, 1, 0, 2, 1, 2, 0.75, 3.0),
    "gc7": (1, 7, 6, 2, 7, 5, 3, 1, 2, 2, 0, 2, 1, 1.5, 3.0),
    "internimage_h": (1, 64, 80, 10, 32, 3, 3, 1, 1, 1, 1, 1, 1, 1.0, 4.0),   # InternImage-H stage 1: 320 = 10 x 32
}


class Dcn:
    def __init__(self, N, H, W, G, C, kh, kw, sh, sw, ph, pw, dh, dw, scale, amp):
        self.N, self.H, self.W, self.G, self.C = N, H, W, G, C
        self.kh, self.kw, self.sh, self.sw, self.ph, self.pw, self.dh, self.dw = kh, kw, sh, sw, ph, pw, dh, dw
        self.scale, self.amp = scale, amp
        self.Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
        self.Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
        self.K = kh * kw

    def args(self):
        return (self.N, self.H, self.W, self.Ho, self.Wo, self.G, self.C, self.kh, self.kw, self.sh, self.sw, self.ph,
                self.pw, self.dh, self.dw, float(self.scale))

    def inputs(self, seed):
        g = gen(seed)
        inp = torch.randn(self.N, self.H, self.W, self.G * self.C, device=DEV, generator=g)
        inp = inp * torch.exp2(torch.randint(-5, 6, (self.N, self.H, self.W, self.G, 1), device=DEV,
                                             generator=g).float()).repeat_interleave(self.C, -1).view_as(inp)
        off = (torch.rand(self.N, self.Ho, self.Wo, self.G * self.K * 2, device=DEV, generator=g) - 0.5) * self.amp
        m = torch.softmax(torch.randn(self.N, self.Ho, self.Wo, self.G, self.K, device=DEV, generator=g), -1)
        return inp.contiguous(), off.contiguous(), m.reshape(self.N, self.Ho, self.Wo, -1).contiguous()


def dcn_fwd(d, inp, off, m, flags=0, iptr=None):
    o = Out((d.N, d.Ho, d.Wo, d.G * d.C))
    assert _lib.lib().vllm_dcnv3_forward_f32(iptr or inp.data_ptr(), off.data_ptr(), m.data_ptr(), o.view.data_ptr(),
                                             *d.args(), flags, stream()) == 0
    return o.check(f"dcnv3 flags={flags}")


def dcn_bwd(d, inp, off, m, go):
    gi, goff, gm = Out(inp.shape, fill=0.0), Out(off.shape), Out(m.shape)
    assert _lib.lib().vllm_dcnv3_backward_f32(inp.data_ptr(), off.data_ptr(), m.data_ptr(), go.data_ptr(),
                                              gi.view.data_ptr(), goff.view.data_ptr(), gm.view.data_ptr(),
                                              *d.args(), stream()) == 0
    return gi.check("grad_input"), goff.check("grad_offset"), gm.check("grad_mask")


def dcn_geom(d, off):
    """(h_low, w_low, mask, lh, lw) [N, Ho, Wo, G, K] by dcn_geom's fp32 sequence; taps kernel_w-major."""
    o = off.view(d.N, d.Ho, d.Wo, d.G, d.K, 2)
    k = torch.arange(d.K, device=DEV)
    i, j = (k // d.kh).float(), (k % d.kh).float()                              # i: column tap, j: row tap
    s = torch.tensor(d.scale, dtype=torch.float32, device=DEV)
    hw_, hh_ = (d.dw * (d.kw - 1)) >> 1, (d.dh * (d.kh - 1)) >> 1
    ow = torch.arange(d.Wo, device=DEV).view(1, 1, d.Wo, 1, 1)
    oh = torch.arange(d.Ho, device=DEV).view(1, d.Ho, 1, 1, 1)
    p0w = (hw_ - d.pw + ow * d.sw).float() - torch.tensor(float(hw_), device=DEV) * s
    p0h = (hh_ - d.ph + oh * d.sh).float() - torch.tensor(float(hh_), device=DEV) * s
    lw_ = p0w + torch.mul(torch.add(i * d.dw, o[..., 0]), s)
    lh_ = p0h + torch.mul(torch.add(j * d.dh, o[..., 1]), s)
    inr = (lh_ > -1) & (lw_ > -1) & (lh_ < d.H) & (lw_ < d.W)
    hf, wf = torch.floor(lh_), torch.floor(lw_)
    lh = torch.where(inr, lh_ - hf, 0.0)
    lw = torch.where(inr, lw_ - wf, 0.0)
    hl, wl = torch.where(inr, hf.long(), 0), torch.where(inr, wf.long(), 0)
    mk = inr.int()
    mk |= (inr & (hl >= 0) & (wl >= 0)).int() << 1
    mk |= (inr & (hl >= 0) & (wl + 1 <= d.W - 1)).int() << 2
    mk |= (inr & (hl + 1 <= d.H - 1) & (wl >= 0)).int() << 3
    mk |= (inr & (hl + 1 <= d.H - 1) & (wl + 1 <= d.W - 1)).int() << 4
    return hl, wl, mk, lh, lw


def dcn_ref(d, inp, off, m, go=None):
    """Forward (z, A) [N, Ho, Wo, G*C]; with go also the backward's z / sum-|term| / hits."""
    hl, wl, mk, lh, lw = dcn_geom(d, off)
    N, Ho, Wo, G, K, C = d.N, d.Ho, d.Wo, d.G, d.K, d.C
    b = torch.arange(N, device=DEV).view(N, 1, 1, 1, 1)
    gg = torch.arange(G, device=DEV).view(1, 1, 1, G, 1)
    base = ((b * d.H + hl) * d.W + wl) * G + gg
    v = inp.double().reshape(-1, C)
    a = m.double().view(N, Ho, Wo, G, K)
    shp = (N, Ho, Wo, G, K, 1)
    z = torch.zeros(N, Ho, Wo, G, C, dtype=torch.float64, device=DEV)
    A = torch.zeros_like(z)
    if go is not None:
        gr = go.double().view(N, Ho, Wo, G, 1, C)
        gi, giA = torch.zeros_like(v), torch.zeros_like(v)
        hits = torch.zeros(v.shape[0], dtype=torch.float64, device=DEV)
        zs = {k: torch.zeros(N, Ho, Wo, G, K, dtype=torch.float64, device=DEV) for k in ("m", "x", "y", "Am", "Ax", "Ay")}
    s = abs(d.scale)
    for (dh, dw, bit), (w, cx, cy) in zip(CORNERS, corner_terms(lh, lw)):
        ok = (mk & bit) != 0
        idx = torch.where(ok, base + (dh * d.W + dw) * G, 0)
        rows = torch.where(ok.view(shp), v[idx.reshape(-1)].view(N, Ho, Wo, G, K, C), 0.0)
        t = torch.where(ok, w * a, 0.0).view(shp) * rows
        z += t.sum(4)
        A += t.abs().sum(4)
        if go is None:
            continue
        vg, vgA = (rows * gr).sum(-1), (rows.abs() * gr.abs()).sum(-1)
        zs["m"] += torch.where(ok, w * vg, 0.0)
        zs["Am"] += torch.where(ok, w.abs() * vgA, 0.0)
        zs["x"] += torch.where(ok, d.scale * a * cx * vg, 0.0)
        zs["Ax"] += torch.where(ok, s * (a * cx).abs() * vgA, 0.0)
        zs["y"] += torch.where(ok, d.scale * a * cy * vg, 0.0)
        zs["Ay"] += torch.where(ok, s * (a * cy).abs() * vgA, 0.0)
        sel = ok.reshape(-1)
        tg = (torch.where(ok, w * a, 0.0).view(shp) * gr).reshape(-1, C)[sel]
        gi.index_add_(0, idx.reshape(-1)[sel], tg)
        giA.index_add_(0, idx.reshape(-1)[sel], tg.abs())
        hits.index_add_(0, idx.reshape(-1)[sel], torch.ones(int(sel.sum()), dtype=torch.float64, device=DEV))
    fwd = (z.view(N, Ho, Wo, G * C), A.view(N, Ho, Wo, G * C))
    if go is None:
        return fwd
    sh = inp.shape
    return fwd, (gi.view(sh), giA.view(sh), hits.view(N, d.H, d.W, G, 1).expand(N, d.H, d.W, G, C).reshape(sh),
                 torch.stack((zs["x"], zs["y"]), -1).view(off.shape), torch.stack((zs["Ax"], zs["Ay"]), -1).view(off.shape),
                 zs["m"].view(m.shape), zs["Am"].view(m.shape))


@pytest.mark.parametrize("case", list(DCN_CASES))
def test_dcnv3_vs_fp64(case):
    """Fast and strict forward and the backward against fp64 on non-square kernels, strides, pads and dilations with
    offset_scale != 1; the fast kernel is taken exactly when C == 32 and K <= 32 (else it is the strict kernel's bits);
    image b of the batch == the image alone; a misaligned input view takes the strict kernel."""
    d = Dcn(*DCN_CASES[case])
    inp, off, m = d.inputs(seed=d.K + d.C)
    go = torch.randn(d.N, d.Ho, d.Wo, d.G * d.C, device=DEV, generator=gen(4))
    (z, A), (zgi, Agi, hits, zgo, Ago, zgm, Agm) = dcn_ref(d, inp, off, m, go)
    strict = dcn_fwd(d, inp, off, m, flags=1)
    within(strict, z, g_(d.K + 3 + 5) * A, "dcnv3_fwd_strict", case)
    fast = dcn_fwd(d, inp, off, m)
    if d.C == 32 and d.K <= 32:
        within(fast, z, g_(d.K + 2 + 4) * A, "dcnv3_fwd_fast", case)
    else:
        assert same_bits(fast, strict), f"{case}: not the strict kernel"
    for b in range(d.N):
        one = (inp[b:b + 1].contiguous(), off[b:b + 1].contiguous(), m[b:b + 1].contiguous())
        d1 = Dcn(1, *DCN_CASES[case][1:])
        assert same_bits(dcn_fwd(d1, *one), fast[b:b + 1]), f"{case}: image {b} != the image alone"
    buf = torch.empty(inp.numel() + 1, device=DEV)
    buf[1:] = inp.flatten()
    assert same_bits(dcn_fwd(d, inp, off, m, iptr=buf[1:].data_ptr()), strict), f"{case}: misaligned != strict"
    gi, goff, gm = dcn_bwd(d, inp, off, m, go)
    within(gi, zgi, g_(hits + 5) * Agi, "dcnv3_bwd_grad_input", case)
    c = -(-d.C // 32) + 5 + 8
    within(goff, zgo, g_(c) * Ago, "dcnv3_bwd_grad_offset", case)
    within(gm, zgm, g_(c) * Agm, "dcnv3_bwd_grad_mask", case)
    _, goff2, gm2 = dcn_bwd(d, inp, off, m, go)
    assert same_bits(goff, goff2) and same_bits(gm, gm2), f"{case}: grad_offset / grad_mask not reproducible"


def test_dcnv3_batch_over_65535_takes_the_strict_kernel():
    d = Dcn(65536, 2, 3, 1, 32, 1, 3, 1, 1, 0, 1, 1, 1, 1.0, 2.0)
    inp, off, m = d.inputs(seed=3)
    z, A = dcn_ref(d, inp, off, m)
    y = dcn_fwd(d, inp, off, m)
    assert same_bits(y, dcn_fwd(d, inp, off, m, flags=1))
    within(y, z, g_(d.K + 3 + 5) * A, "dcnv3_fwd_strict", "N = 65536")


# ---------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------
def test_rejections_leave_every_output_untouched():
    lib, st = _lib.lib(), stream()
    pyr = Pyr([(4, 4)] * 9)                                                       # 9 levels: more than 8
    v = torch.zeros(1, pyr.S, 2, 32, device=DEV)
    vb = v.bfloat16()
    loc = torch.zeros(1, 3, 2, 9, 4, 2, device=DEV)
    aw = torch.zeros(1, 3, 2, 9, 4, device=DEV)
    o32, o16 = Out((1, 3, 64)), Out((1, 3, 64), torch.bfloat16)
    gv, gl, ga = Out(v.shape), Out(loc.shape), Out(aw.shape)
    P_, V, V16, LO, A_ = pyr.dev.data_ptr(), v.data_ptr(), vb.data_ptr(), loc.data_ptr(), aw.data_ptr()
    S, lsi, H = pyr.S, pyr.lsi.data_ptr(), pyr.host.data_ptr()

    def f32(vp=V, o=o32.view.data_ptr(), N=1, M=2, D=32, L=1, P=4, lp=LO):
        return lib.vllm_msda_forward_f32(vp, P_, lsi, lp, A_, o, N, S, M, D, L, 3, P, H, 0, st)

    def bf16(vp=V16, o=o16.view.data_ptr(), N=1, M=2, D=32, L=1, P=4, lp=LO):
        return lib.vllm_msda_forward_bf16v(vp, P_, lsi, lp, A_, o, 1, N, S, M, D, L, 3, P, H, st)

    def f64(N=1, M=2, L=1):
        return lib.vllm_msda_forward_f64(V, P_, lsi, LO, A_, o32.view.data_ptr(), N, S, M, 32, L, 3, 4, st)

    def bwd(N=1, M=2, L=1):
        return lib.vllm_msda_backward_f32(V, P_, lsi, LO, A_, V, gv.view.data_ptr(), gl.view.data_ptr(),
                                          ga.view.data_ptr(), N, S, M, 32, L, 3, 4, st)

    def fused(L=4, P=4, D=32):
        return lib.vllm_msda_forward_fused_bf16(V16, lsi, V16, 2 * 16 * 3, LO, o16.view.data_ptr(), 1, None, 1, S, 2, D,
                                                L, S, P, H, st)

    cases = {
        "bf16v D=16": (bf16(D=16), EUNSUPPORTED), "bf16v L=9": (bf16(L=9), EUNSUPPORTED),
        "bf16v K=33": (bf16(L=3, P=11), EUNSUPPORTED),
        "bf16v value misaligned": (bf16(vp=V16 + 2), EALIGN), "bf16v out misaligned": (bf16(o=o16.view.data_ptr() + 2), EALIGN),
        "bf16v loc misaligned": (bf16(lp=LO + 4), EALIGN),
        "fused L=3": (fused(L=3), EUNSUPPORTED), "fused P=2": (fused(P=2), EUNSUPPORTED), "fused D=16": (fused(D=16), EUNSUPPORTED),
        "f32 L=9": (f32(L=9), EUNSUPPORTED), "f64 L=9": (f64(L=9), EUNSUPPORTED), "bwd L=9": (bwd(L=9), EUNSUPPORTED),
        "bf16v L=9 P=1": (bf16(L=9, P=1), EUNSUPPORTED),
        "f32 N<0": (f32(N=-1), EINVAL), "f32 M=0": (f32(M=0), EINVAL), "f32 P=0": (f32(P=0), EINVAL),
        "bf16v N<0": (bf16(N=-1), EINVAL), "f64 N<0": (f64(N=-1), EINVAL), "bwd N<0": (bwd(N=-1), EINVAL),
        "bwd M=0": (bwd(M=0), EINVAL),
    }
    d = Dcn(1, 6, 6, 1, 32, 3, 3, 1, 1, 1, 1, 1, 1, 1.0, 1.0)
    inp, off, m = d.inputs(seed=1)
    od, gi, goff, gm = Out((1, 6, 6, 32)), Out(inp.shape), Out(off.shape), Out(m.shape)
    a = list(d.args())
    for i, name in ((0, "N"), (1, "H_in"), (5, "group"), (6, "group_channels"), (7, "kernel_h"), (10, "stride_w"),
                    (14, "dilation_w")):
        bad = a.copy()
        bad[i] = -1 if i == 0 else 0
        cases[f"dcnv3 fwd {name}"] = (lib.vllm_dcnv3_forward_f32(inp.data_ptr(), off.data_ptr(), m.data_ptr(),
                                                                 od.view.data_ptr(), *bad, 0, st), EINVAL)
        cases[f"dcnv3 bwd {name}"] = (lib.vllm_dcnv3_backward_f32(inp.data_ptr(), off.data_ptr(), m.data_ptr(), od.view.data_ptr(),
                                                                  gi.view.data_ptr(), goff.view.data_ptr(), gm.view.data_ptr(),
                                                                  *bad, st), EINVAL)
    torch.cuda.synchronize()
    for what, (rc, want) in cases.items():
        assert rc == want, f"{what}: returned {rc}, documented {want}"
    for o in (o32, o16, gv, gl, ga, od, gi, goff, gm):
        assert o.untouched(), "a rejected call wrote to its outputs"
