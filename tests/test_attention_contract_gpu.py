"""GPU: every attention path (csrc/attention.cu, csrc/attention_wgmma.cu) against a float64 reference of the same op on
the same bf16 inputs, exact key-count probes of its index logic, the split-KV path at forced split counts, and the
bit-identities and memory rules that tie its entry points together.

Paths: the wgmma kernel (head_dim 128 / 256 without attn_mask / attn_bias, the default variant), the warp-MMA kernel
(every head_dim; `ATTN_WARP_MMA` forces it), the one-warp-per-window Swin kernel (head_dim 32, attn_bias only,
Tq == Tk <= 64), the live-tile walk of a sparse attn_mask, and the split-KV partials + combine of both families.

1. Numerics.  The reference takes the bf16 q / k / v (and fp32 bias), forms s = scale * q @ k^T (+ bias) in float64,
   applies every mask as -inf, P = softmax(s), ref = P @ V; a row that can attend no key has ref = 0.  Per row i:
       |out - ref| <= 2^-8 |ref| + (1 + 2^-6) * (2^-8 + 2 D_i + ceil(Tk / 16) 2^-22) * (P @ |V|)_i
       D_i = ceil(D / 16) 2^-24 scale max_j (|q_i| @ |k_j|^T) + 2^-21 max_j |s_ij|      (j over the keys row i attends)
   - 2^-8 |ref|: the output is rounded to bf16, whose unit roundoff is 2^-8 (8 significant bits); the (1 + 2^-6) on
     the other terms covers that rounding applied to their error.
   - 2^-8 (P @ |V|): P is rounded to bf16 before P @ V, while the row sum l adds the unrounded fp32 p, so the
     rounding of each p does not cancel in O / l.
   - 2 D_i (P @ |V|): a score error d moves p by the factor e^d, once in O and once in l.  The fp32 accumulation of q.k
     over D (bf16 products are exact; one rounding of the sum of magnitudes per k16 step), and in the log2 domain the
     rounding of scale * log2(e), of the product, of the FMA with the row max and of the bias FMA, each relative to
     |s| or the row max (2^-21 allows eight).  The error of ex2.approx / exp2f (about 2^-22 relative) is inside the
     2^-6 margin.
   - ceil(Tk / 16) 2^-22 (P @ |V|): the fp32 accumulation of O (one rounding per k16 step), the per-tile rescales,
     and the split-KV combine (exp2f of the partial maxima, the sum over splits).
   There is no max|ref| term: a dropped rescale, a key off by one at the causal diagonal or a wrong slab of a mask
   moves rows whose P @ |V| is small far outside it.  Inputs: "peaked" (score std ~3), "wide" (scale 4 / sqrt(D),
   score spread > 64 per row) and "rising" (a ramp on one k column raises the row max by ~3 per 64-key tile, so every
   tile rescales O and l by corr < 1).  The worst err / bound is 0.84 over the cases of 1 and 0.67 over the split
   counts of 3 (NVIDIA H100 80GB HBM3, 700 W power limit): the 2^-8 terms are nearly reached, so a bound built on
   half that rounding fails.  `pytest -rP` prints it per case.

2. Probes.  q = 0 makes every attendable score exactly 0, every p exactly 1 (ex2(0) = exp2f(0) = 1) and every masked p
   exactly 0, and V is a 0 / 1 fingerprint: v[b, j, hkv, c] = 1 iff (7 j + 3 hkv + 5 b) mod D == c.  Then
   O[b, i, h, c] = n (the attendable keys of row i that carry column c's fingerprint) and l = N (all of them), both
   exact in fp32, so the output is exactly bf16(n * fl(1 / N)) (0 for N = 0), bit for bit.  One key dropped, counted
   twice or read from the wrong batch entry / kv head changes n or N and with it the bytes.  Masks in attn_bias are
   0 / -inf here.

3. Split-KV at forced counts (`vllm_attention_set_splits`) 1 / 2 / 3 / 7 / 64 on both families, head_dim 32 / 128 /
   256, with key masks, seqlens that leave whole splits empty, and causal: within the bound of 1, exactly the probe
   of 2, and the partials use exactly the first batch * heads * n * Tq * (D + 2) floats of a NaN-filled workspace.

Every call writes into a NaN-filled [B, Tq, H * D] view with a row pitch larger than H * D inside a sentinel-filled
buffer with 8 spare rows below each batch entry: every element of the view must be written and no sentinel changed.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from visionllm_b200 import _lib  # noqa: E402

VARIANTS = {"default": _lib.ATTN_DEFAULT, "warp_mma": _lib.ATTN_WARP_MMA}   # default: wgmma / window kernel
SENTINEL = 4320.0                            # exact in bf16; the kernels never write it here
SPLITS = (1, 2, 3, 7, 64)
NAN_ROWS = 128                               # NaN rows after the last key of every batch entry of a K / V buffer


def ops():
    from visionllm_b200 import ops as o
    return o


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------
# calls
# ---------------------------------------------------------------------------------------------------------------------
def out_buffer(B, Tq, HD):
    """A sentinel-filled [B, Tq + 8, HD + 64] bf16 buffer and its NaN-filled [B, Tq, HD] view."""
    buf = torch.full((B, Tq + 8, HD + 64), SENTINEL, dtype=torch.bfloat16, device="cuda")
    view = buf[:, :Tq, :HD]
    view.fill_(float("nan"))
    return buf, view


def check_written(buf, view, what):
    B, Tq, HD = view.shape
    assert not view.isnan().any(), \
        f"{what}: {int(view.isnan().sum())} output elements are NaN (never written, or a read past the inputs)"
    inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    inside[:, :Tq, :HD] = True
    assert (buf[~inside] == SENTINEL).all(), f"{what}: a store landed outside [B, Tq, H*D]"


def workspace(p, n):
    """A NaN-filled fp32 workspace with 4096 floats more than n splits need, and the number they need."""
    B, Tq, H, D = p["q"].shape
    need = B * H * n * Tq * (D + 2)
    return torch.full((need + 4096,), float("nan"), dtype=torch.float32, device="cuda"), need


def raw(p, out, ws=None, ws_bytes=0, scale=None):
    """vllm_attention_bf16 itself: ws None = a NULL workspace (no split)."""
    q, k, v = p["q"], p["k"], p["v"]
    B, Tq, H, D = q.shape
    Tk, Hkv = k.shape[1], k.shape[2]
    ptr = lambda t: None if t is None else t.data_ptr()        # noqa: E731
    bias = p.get("bias")
    return _lib.lib().vllm_attention_bf16(
        q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, Tq, Tk, H, Hkv, D,
        q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0), out.stride(1),
        ptr(p.get("seqlens")), ptr(p.get("key_mask")), ptr(p.get("attn_mask")), ptr(bias),
        0 if bias is None else bias.shape[0], int(p.get("causal", False)), float(p["scale"] if scale is None else scale),
        ptr(ws), ws_bytes, torch.cuda.current_stream().cuda_stream)


def attend(p, variant, splits=None, via_ops=False, what=""):
    """One call on `variant` into a sentinel-padded output view.  splits None: a NULL workspace; n: the count forced to
    n with a workspace of exactly n partials, whose use is checked; via_ops: ops.attention and its own workspace."""
    B, Tq, H, D = p["q"].shape
    buf, out = out_buffer(B, Tq, H * D)
    with _lib.knob("attention_set_variant", VARIANTS[variant]):
        if via_ops or "tiles" in p:
            ops().attention(p["q"], p["k"], p["v"], causal=p.get("causal", False), scale=p["scale"],
                            seqlens=p.get("seqlens"), key_mask=p.get("key_mask"),
                            attn_mask=p.get("tiles", p.get("attn_mask")), attn_bias=p.get("bias"), out=out)
        elif splits is None:
            assert raw(p, out) == 0, what
        else:
            ws, need = workspace(p, splits)
            with _lib.knob("attention_set_splits", splits):
                assert raw(p, out, ws, need * 4) == 0, what
            used = need if splits > 1 else 0
            assert not ws[:used].isnan().any(), f"{what}: {int(ws[:used].isnan().sum())} partial floats not written"
            assert bits(ws[used:]).eq(bits(ws[-1:])).all(), f"{what}: the workspace was written past {splits} partials"
    torch.cuda.synchronize()
    check_written(buf, out, what)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------
def fingerprint(B, Tk, Hkv, D):
    j = torch.arange(Tk, device="cuda")[None, :, None]
    h = torch.arange(Hkv, device="cuda")[None, None, :]
    b = torch.arange(B, device="cuda")[:, None, None]
    return torch.nn.functional.one_hot((7 * j + 3 * h + 5 * b) % D, D).bfloat16()


def group_mask(B, H, T, group, g):
    """UniPose's keypoint-decoder mask: groups attend within themselves plus a few off-diagonal stripes, one query row
    that attends nothing, one query block without a live tile."""
    idx = torch.arange(T, device="cuda")
    allow = ((idx[:, None] // group) == (idx[None, :] // group))[None].repeat(B * H, 1, 1)
    n_groups = (T + group - 1) // group
    for bh in range(B * H):
        for _ in range(2):
            gi, gj = (int(x) for x in torch.randint(0, n_groups, (2,), device="cuda", generator=g))
            allow[bh, gi * group:(gi + 1) * group, gj * group] = True
    allow[0, 5] = False
    allow[-1, 64:128] = False
    return allow


def build(s, D, kind, seed=0):
    """The problem of spec `s` at head_dim D with inputs of `kind` ("peaked", "wide", "rising" or "probe")."""
    B, Tq, Tk, H = s["B"], s["Tq"], s["Tk"], s["H"]
    Hkv = s.get("Hkv", H)
    g = gen(seed + 1000 * D + Tq + 7 * Tk)
    scale = s.get("scale", 1.0) * D ** -0.5 * (4.0 if kind == "wide" else 1.0)
    p = dict(scale=scale, causal=s.get("causal", False))
    if kind == "probe":
        q = torch.zeros(B, Tq, H, D, device="cuda", dtype=torch.bfloat16)
        k = torch.randn(B, Tk, Hkv, D, device="cuda", generator=g).bfloat16()
        v = fingerprint(B, Tk, Hkv, D)
    else:
        a = {"peaked": 3 ** 0.5, "wide": 2.0, "rising": 1.0}[kind]
        q = torch.randn(B, Tq, H, D, device="cuda", generator=g) * a
        k = torch.randn(B, Tk, Hkv, D, device="cuda", generator=g) * a
        if kind == "rising":
            q[..., 0] = 4.0
            k[..., 0] += torch.arange(Tk, device="cuda")[None, :, None] * (3.0 / (64 * scale * 4.0))
        q, k = q.bfloat16(), k.bfloat16()
        v = torch.randn(B, Tk, Hkv, D, device="cuda", generator=g).bfloat16()
    p.update(q=q, k=k, v=v)
    if "seqlens" in s:
        p["seqlens"] = torch.tensor(s["seqlens"], dtype=torch.int32, device="cuda")
    if s.get("key_mask"):
        km = torch.rand(B, Tk, device="cuda", generator=g) > 0.3
        km[0] = True
        if Tk >= 192:
            km[1, 64:128] = False                                   # a fully masked 64-key tile
        km[-1] = False                                              # a batch entry that attends nothing
        p["key_mask"] = km.view(torch.uint8)
    if s.get("attn_mask"):
        am = torch.rand(B * H, Tq, Tk, device="cuda", generator=g) > 0.5
        am[-1, Tq // 2] = False                                     # a row that attends nothing
        p["attn_mask"] = am.view(torch.uint8)
    if "nB" in s:
        shape = (s["nB"], H, Tq, Tk)
        if kind == "probe":                                         # masks as 0 / -inf
            bias = torch.where(torch.rand(shape, device="cuda", generator=g) > 0.4, 0.0, float("-inf"))
            bias[-1, -1, Tq // 2] = float("-inf")                   # a row that attends nothing
        else:
            bias = torch.randn(shape, device="cuda", generator=g) * 2
            bias[torch.rand(shape, device="cuda", generator=g) < 0.1] = -100.0
        p["bias"] = bias
    if "group" in s:
        p["attn_mask"] = group_mask(B, H, Tq, s["group"], g).view(torch.uint8)
        p["tiles"] = ops().attention_mask_tiles(p["attn_mask"])
    return p


def allowed(p):
    """[B, H, Tq, Tk]: which keys each query row attends."""
    B, Tq, H, _ = p["q"].shape
    Tk = p["k"].shape[1]
    i = torch.arange(Tq, device="cuda")[:, None]
    j = torch.arange(Tk, device="cuda")[None, :]
    a = torch.ones(B, H, Tq, Tk, dtype=torch.bool, device="cuda")
    if p.get("causal"):
        a &= j <= i + (Tk - Tq)
    if p.get("seqlens") is not None:
        a &= j < p["seqlens"].long()[:, None, None, None]
    if p.get("key_mask") is not None:
        a &= p["key_mask"].bool()[:, None, None, :]
    if p.get("attn_mask") is not None:
        a &= p["attn_mask"].bool().view(B, H, Tq, Tk)
    if p.get("bias") is not None:
        a &= p["bias"][torch.arange(B, device="cuda") % p["bias"].shape[0]] != float("-inf")
    return a


def per_head(t, H):
    """[B, T, Hkv, D] -> float64 [B, H, T, D], kv heads repeated for grouped-query attention."""
    return t.double().permute(0, 2, 1, 3).repeat_interleave(H // t.shape[2], 1)


def reference(p):
    """float64 output and the bound of the module docstring, both [B, Tq, H * D]."""
    B, Tq, H, D = p["q"].shape
    Tk = p["k"].shape[1]
    q, k, v = per_head(p["q"], H), per_head(p["k"], H), per_head(p["v"], H)
    allow = allowed(p)
    s = p["scale"] * (q @ k.transpose(-1, -2))
    if p.get("bias") is not None:
        s = s + p["bias"].double()[torch.arange(B, device="cuda") % p["bias"].shape[0]]
    s = s.masked_fill(~allow, float("-inf"))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    P = e / torch.where(l > 0, l, torch.ones_like(l))
    ref, pav = P @ v, P @ v.abs()
    qk = (p["scale"] * (q.abs() @ k.abs().transpose(-1, -2))).masked_fill(~allow, 0).amax(-1, keepdim=True)
    smax = s.abs().masked_fill(~allow, 0).amax(-1, keepdim=True)
    delta = math.ceil(D / 16) * 2.0 ** -24 * qk + 2.0 ** -21 * smax
    bound = 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -6) * (2.0 ** -8 + 2 * delta + math.ceil(Tk / 16) * 2.0 ** -22) * pav
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B, Tq, H * D)   # noqa: E731
    return flat(ref), flat(bound)


def probe_expect(p):
    """bf16(n * fl(1 / N)) of the module docstring, computed in IEEE fp32 on the CPU."""
    B, Tq, H, D = p["q"].shape
    a = allowed(p).double()
    n = (a @ per_head(p["v"], H)).float().cpu()
    N = a.sum(-1, keepdim=True).float().cpu()
    out = torch.where(N > 0, n * (1.0 / N), torch.zeros_like(n)).bfloat16()
    return out.permute(0, 2, 1, 3).reshape(B, Tq, H * D).cuda()


def check_fp64(out, ref, bound, what):
    err = (out.double() - ref).abs()
    bad = err > bound
    ratio = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    i = int(ratio.argmax())
    assert not bad.any(), (f"{what}: {int(bad.sum())} / {err.numel()} outside the bound; worst at "
                           f"{i}: out {out.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r} "
                           f"bound {bound.flatten()[i].item():.3g}")
    return float(ratio.flatten()[i])


def check_probe(out, expect, what):
    diff = bits(out) != bits(expect)
    assert not diff.any(), (f"{what}: {int(diff.sum())} / {diff.numel()} elements differ from the exact key count; "
                            f"first at {tuple(int(x) for x in diff.nonzero()[0])}")


def variants_of(s, D):
    """The variants that run a different kernel for this call (the default is the warp-MMA kernel itself elsewhere)."""
    if s.get("attn_mask") or "group" in s:
        return ["warp_mma"]
    if "nB" in s:
        window = D == 32 and s["Tq"] == s["Tk"] <= 64 and not s.get("causal") and "seqlens" not in s
        return ["default", "warp_mma"] if window else ["warp_mma"]
    return ["default", "warp_mma"] if D in (128, 256) else ["warp_mma"]


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2: every path against fp64 and the exact probe
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    "vit_1025": dict(B=2, Tq=1025, Tk=1025, H=2, kinds=("wide",)),          # InternViT tile
    "llm_causal": dict(B=1, Tq=1536, Tk=1536, H=2, causal=True),
    "causal_q1": dict(B=2, Tq=1, Tk=300, H=2, causal=True),
    "causal_q65": dict(B=1, Tq=65, Tk=700, H=2, causal=True),
    "causal_q_gt_k": dict(B=2, Tq=200, Tk=70, H=2, causal=True),             # rows < 130 attend nothing
    "gqa_8_2": dict(B=2, Tq=200, Tk=333, H=8, Hkv=2),
    "seqlens": dict(B=4, Tq=130, Tk=300, H=2, seqlens=[300, 0, 17, 129], scale=0.7),
    "gdino_v2t": dict(B=3, Tq=900, Tk=80, H=4, key_mask=True),               # vision queries over text keys
    "gdino_t2v": dict(B=3, Tq=80, Tk=4352, H=4, key_mask=True, kinds=("wide",)),
    "attn_mask": dict(B=2, Tq=100, Tk=150, H=3, attn_mask=True),
    "attn_bias": dict(B=4, Tq=90, Tk=130, H=3, nB=2),
}
WINDOW = {f"window_T{T}_nB{nB}": dict(B=8, Tq=T, Tk=T, H=3, nB=nB) for T in (1, 16, 49, 64) for nB in (1, 4)}
ALL_CASES = [(c, D) for c in CASES for D in (32, 64, 128, 256)] + [(c, 32) for c in WINDOW] + [("live_tiles", 32)]
SPECS = dict(CASES, **WINDOW, live_tiles=dict(B=1, Tq=690, Tk=690, H=2, group=69))


@pytest.mark.parametrize("case,D", ALL_CASES, ids=[f"{c}-D{D}" for c, D in ALL_CASES])
def test_every_path_vs_fp64_and_exact_probe(case, D):
    """Each case on every kernel that takes it, through vllm_attention_bf16 with a NULL workspace and through
    ops.attention (which passes a workspace to few-query calls): within the fp64 bound for each input kind, and the
    probe's exact bytes."""
    s = SPECS[case]
    worst = 0.0
    for kind in ("peaked", "rising") + s.get("kinds", ()):
        p = build(s, D, kind)
        ref, bound = reference(p)
        for variant in variants_of(s, D):
            for via_ops in (False, True):
                what = f"{case} D={D} {kind} {variant} {'ops.attention' if via_ops else 'no split'}"
                worst = max(worst, check_fp64(attend(p, variant, via_ops=via_ops, what=what), ref, bound, what))
    p = build(s, D, "probe")
    expect = probe_expect(p)
    for variant in variants_of(s, D):
        for via_ops in (False, True):
            what = f"{case} D={D} probe {variant} {'ops.attention' if via_ops else 'no split'}"
            check_probe(attend(p, variant, via_ops=via_ops, what=what), expect, what)
    print(f"worst err/bound {worst:.4f}")


# ---------------------------------------------------------------------------------------------------------------------
# 3: split-KV at every forced count
# ---------------------------------------------------------------------------------------------------------------------
SPLIT_CASES = {
    "plain": dict(B=2, Tq=80, Tk=1000, H=2),
    "key_mask": dict(B=3, Tq=80, Tk=1000, H=2, key_mask=True),
    "seqlens": dict(B=3, Tq=80, Tk=1000, H=2, seqlens=[1000, 100, 0]),     # splits with no key tile; all of them
    "causal": dict(B=1, Tq=200, Tk=600, H=2, causal=True),
}
FAMILIES = [("warp_mma", 32), ("warp_mma", 128), ("warp_mma", 256), ("default", 128), ("default", 256)]


@pytest.mark.parametrize("case", list(SPLIT_CASES))
@pytest.mark.parametrize("variant,D", FAMILIES, ids=[f"{v}-D{D}" for v, D in FAMILIES])
def test_split_kv_every_count(variant, D, case):
    """n = 1 / 2 / 3 / 7 / 64 splits: within the fp64 bound, the probe's exact bytes, and exactly n partials of the
    workspace written (n = 1: none)."""
    s = SPLIT_CASES[case]
    p = build(s, D, "peaked")
    ref, bound = reference(p)
    pp = build(s, D, "probe")
    expect = probe_expect(pp)
    worst = 0.0
    for n in SPLITS:
        what = f"{case} {variant} D={D} splits={n}"
        worst = max(worst, check_fp64(attend(p, variant, splits=n, what=what), ref, bound, what))
        check_probe(attend(pp, variant, splits=n, what=what + " probe"), expect, what + " probe")
    print(f"worst err/bound {worst:.4f}")


# ---------------------------------------------------------------------------------------------------------------------
# 4: bit-identities (NULL workspace unless stated)
# ---------------------------------------------------------------------------------------------------------------------
IDENT = [("default", 128), ("default", 256), ("warp_mma", 64), ("warp_mma", 128), ("warp_mma", 256)]


def nan_tailed(t, extra=NAN_ROWS):
    """t [B, T, h, D] copied into a NaN-filled [B, T + extra, h, D] buffer: a read past row T poisons the result."""
    buf = torch.full((t.shape[0], t.shape[1] + extra) + tuple(t.shape[2:]), float("nan"), dtype=t.dtype, device="cuda")
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


@pytest.mark.parametrize("variant,D", IDENT, ids=[f"{v}-D{D}" for v, D in IDENT])
def test_slices_and_batch_entries_equal_the_full_call(variant, D):
    """Query-row slices [a:b] (non-causal) and suffixes [a:Tq] (causal: the diagonal moves into other query tiles, and
    the tiles it masks fully must leave the online state untouched) equal the full call; one batch entry alone equals
    that entry of the batched call, with seqlens and with a key mask."""
    s = dict(B=3, Tq=333, Tk=333, H=2)
    p = build(s, D, "peaked")
    full = attend(p, variant)
    for a, b in ((0, 1), (70, 200), (129, 333)):
        assert same_bits(attend(dict(p, q=p["q"][:, a:b]), variant), full[:, a:b]), f"rows {a}:{b}"
    pc = dict(p, causal=True)
    full_c = attend(pc, variant)
    for a in (1, 64, 200, 332):
        assert same_bits(attend(dict(pc, q=p["q"][:, a:]), variant), full_c[:, a:]), f"causal rows {a}:"
    km = build(dict(s, key_mask=True), D, "peaked")["key_mask"]
    for extra in (dict(seqlens=torch.tensor([333, 100, 0], dtype=torch.int32, device="cuda")), dict(key_mask=km)):
        pe = dict(p, **extra)
        full_e = attend(pe, variant)
        for b in range(3):
            one = {n: (t[b:b + 1] if n in ("q", "k", "v", "seqlens", "key_mask") else t) for n, t in pe.items()}
            assert same_bits(attend(one, variant), full_e[b:b + 1]), f"batch entry {b} with {list(extra)}"


@pytest.mark.parametrize("variant,D", IDENT, ids=[f"{v}-D{D}" for v, D in IDENT])
def test_gqa_packed_views_and_mask_forms_are_bit_identical(variant, D):
    """GQA == K / V repeat_interleave'd to H heads; packed strided q / k / v == contiguous copies; a key_mask that is a
    length-L prefix == seqlens L; an all-True key_mask == no mask; seqlens Tk and Tk + 70 == no seqlens (K / V followed
    by NaN rows, so a key read past Tk shows); a forced split count with a NULL workspace == no split."""
    B, T, H = 2, 333, 8
    p = build(dict(B=B, Tq=T, Tk=T, H=H, Hkv=2), D, "peaked")
    p["k"], p["v"] = nan_tailed(p["k"]), nan_tailed(p["v"])
    base = attend(p, variant)
    rep = dict(p, k=p["k"].repeat_interleave(4, 2), v=p["v"].repeat_interleave(4, 2))
    assert same_bits(attend(rep, variant), base), "GQA != repeated K / V"
    qkv = torch.full((B, T + NAN_ROWS, 4, H, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    qkv[:, :T, 0], qkv[:, :T, 1], qkv[:, :T, 2] = p["q"], rep["k"], rep["v"]     # slot 3: NaN columns between rows
    packed = dict(p, q=qkv[:, :T, 0], k=qkv[:, :T, 1], v=qkv[:, :T, 2])
    assert same_bits(attend(packed, variant), base), "packed strided views != contiguous"
    L = [T - 100, 17]
    prefix = torch.arange(T, device="cuda")[None, :] < torch.tensor(L, device="cuda")[:, None]
    sl = torch.tensor(L, dtype=torch.int32, device="cuda")
    assert same_bits(attend(dict(p, key_mask=prefix.view(torch.uint8)), variant), attend(dict(p, seqlens=sl), variant)), \
        "prefix key_mask != seqlens"
    ones = torch.ones(B, T, dtype=torch.uint8, device="cuda")
    assert same_bits(attend(dict(p, key_mask=ones), variant), base), "all-True key_mask != no mask"
    for extra in (0, 70):
        sl = torch.full((B,), T + extra, dtype=torch.int32, device="cuda")
        assert same_bits(attend(dict(p, seqlens=sl), variant), base), f"seqlens = Tk + {extra} != no seqlens"
    out = torch.empty(B, T, H * D, dtype=torch.bfloat16, device="cuda")
    with _lib.knob("attention_set_variant", VARIANTS[variant]), _lib.knob("attention_set_splits", 7):
        assert raw(p, out) == 0
    assert same_bits(out, base), "a forced split count with a NULL workspace split the call"


@pytest.mark.parametrize("T", [1, 16, 49, 64])
def test_window_kernel_equals_warp_mma(T):
    """The one-warp-per-window kernel == the warp-MMA kernel on a single key tile, bit for bit, 1 and 4 bias slabs."""
    for nB in (1, 4):
        for kind in ("peaked", "probe"):
            p = build(dict(B=8, Tq=T, Tk=T, H=3, nB=nB), 32, kind)
            assert same_bits(attend(p, "default"), attend(p, "warp_mma")), f"T={T} nB={nB} {kind}"


def test_strided_out_view_equals_fresh_output():
    """ops.attention(out=<view with a row pitch>) == ops.attention() into a fresh tensor, with and without a split."""
    for s, D in ((dict(B=2, Tq=80, Tk=4352, H=4, key_mask=True), 256), (dict(B=2, Tq=300, Tk=300, H=2), 64)):
        p = build(s, D, "peaked")
        fresh = ops().attention(p["q"], p["k"], p["v"], scale=p["scale"], key_mask=p.get("key_mask"))
        assert same_bits(attend(p, "default", via_ops=True), fresh), f"{s}"


# ---------------------------------------------------------------------------------------------------------------------
# 5: memory contract
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,D", IDENT, ids=[f"{v}-D{D}" for v, D in IDENT])
def test_masked_rows_may_hold_any_finite_value(variant, D):
    """K / V rows in [seqlens, Tk) and key-masked rows filled with +-3e38 (finite; the wgmma kernel multiplies masked V
    rows by P = 0, so they must not be NaN / Inf) give the bytes of the call with those rows zero, split or not."""
    B, Tq, Tk, H = 3, 80, 1000, 2
    p = build(dict(B=B, Tq=Tq, Tk=Tk, H=H, key_mask=True, seqlens=[1000, 640, 0]), D, "peaked")
    masked = ~(p["key_mask"].bool() & (torch.arange(Tk, device="cuda")[None, :] < p["seqlens"].long()[:, None]))
    huge = torch.where(torch.rand(B, Tk, H, D, device="cuda", generator=gen(5)) > 0.5, 3e38, -3e38).bfloat16()
    zero = dict(p, k=p["k"].masked_fill(masked[..., None, None], 0), v=p["v"].masked_fill(masked[..., None, None], 0))
    big = dict(p, k=torch.where(masked[..., None, None], huge, p["k"]), v=torch.where(masked[..., None, None], huge, p["v"]))
    for n in (None, 3):
        assert same_bits(attend(big, variant, splits=n), attend(zero, variant, splits=n)), f"splits={n}"


# ---------------------------------------------------------------------------------------------------------------------
# 6: rejections
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,D", [("default", 128), ("warp_mma", 64)])
def test_rejections_leave_the_output_untouched(variant, D):
    """scale 0 / -0.5 / NaN / Inf: VLLM_EINVAL from vllm_attention_bf16 and vllm_attention_bf16_tiles; a workspace one
    float short of the forced split count: VLLM_EINVAL; split counts outside [0, 64] are rejected and change nothing.
    None of them writes the output."""
    p = build(dict(B=2, Tq=80, Tk=600, H=2), D, "peaked")
    B, Tq, H, _ = p["q"].shape
    Tk = p["k"].shape[1]
    buf, out = out_buffer(B, Tq, H * D)
    before = buf.clone()
    L = _lib.lib()
    am = torch.ones(B * H, Tq, Tk, dtype=torch.uint8, device="cuda")
    tiles = ops().attention_mask_tiles(am)
    with _lib.knob("attention_set_variant", VARIANTS[variant]):
        for bad in (0.0, -0.5, float("nan"), float("inf")):
            assert raw(p, out, scale=bad) == -1, f"scale {bad}"
            rc = L.vllm_attention_bf16_tiles(
                p["q"].data_ptr(), p["k"].data_ptr(), p["v"].data_ptr(), out.data_ptr(), B, Tq, Tk, H, H, D,
                p["q"].stride(0), p["q"].stride(1), p["k"].stride(0), p["k"].stride(1), p["v"].stride(0),
                p["v"].stride(1), out.stride(0), out.stride(1), None, None, am.data_ptr(), bad, tiles.counts.data_ptr(),
                tiles.lists.data_ptr(), torch.cuda.current_stream().cuda_stream)
            assert rc == -1, f"tiles, scale {bad}"
        ws, need = workspace(p, 7)
        with _lib.knob("attention_set_splits", 7):
            assert raw(p, out, ws, need * 4 - 4) == -1, "a workspace one float short of 7 partials"
            assert L.vllm_attention_set_splits(-1) == -1 and L.vllm_attention_set_splits(65) == -1
            torch.cuda.synchronize()
            assert same_bits(buf, before), "a rejected call wrote the output"
            assert raw(p, out, ws, need * 4) == 0                   # the count is still 7 ...
        torch.cuda.synchronize()
        assert not ws[:need].isnan().any() and ws[need:].isnan().all()   # ... and exactly 7 partials were written


def test_ops_attention_rejects_a_wrong_out():
    """ops.attention raises on an `out` of the wrong dtype, shape, device, or with a column stride != 1."""
    p = build(dict(B=2, Tq=64, Tk=64, H=2), 64, "peaked")
    B, Tq, H, D = p["q"].shape
    wide = torch.empty(B, Tq, 2 * H * D, dtype=torch.bfloat16, device="cuda")
    bad = {"dtype": torch.empty(B, Tq, H * D, dtype=torch.float32, device="cuda"),
           "shape": torch.empty(B, Tq, H * D + 8, dtype=torch.bfloat16, device="cuda"),
           "stride": wide[:, :, ::2],
           "device": torch.empty(B, Tq, H * D, dtype=torch.bfloat16)}
    for name, out in bad.items():
        before = wide.clone()
        with pytest.raises(RuntimeError):
            ops().attention(p["q"], p["k"], p["v"], out=out)
        torch.cuda.synchronize()
        assert same_bits(wide, before), name
