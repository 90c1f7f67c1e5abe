"""GPU: the glue kernels that decide the model's externally visible integers -- sequence assembly (csrc/seqglue.cu), the
sine position embedding (csrc/posembed.cu), detection top-k and the mask chain (csrc/postproc.cu) and the padded head
stacking of the attention backward (csrc/train_ops.cu) -- against exact and float64 oracles of the same operation on
the same inputs.

Sequence assembly is exact.  `seq_oracle` restates modeling_visionllmv2.py:426-486 (overwrite form: the k-th slot
after a det / seg / grd tool takes [EMB] + k and row k of emb_embeddings_det, after a pose tool of _pose), :582-605
(the k-th <im_patch> slot of the flattened batch takes the k-th row of the tile rows of the samples that have image
tokens) and :776-787 ([EMB] positions per row, in order) as python loops; its CPU self-test pins it to
`ref_emb_overwrite` and to the model's `inject_emb` / `scatter_image_tokens` / `gather_text_query`.  `vllm_seq_index`
must return new_ids, kind, row, emb_count, emb_pos[:count] and status IDENTICAL to it; the single 1024-thread CTA
carries the <im_patch> rank from one 1024-position chunk to the next, so runs straddle chunks with image-less samples
between them.  The row copies (`assemble_embeds`, `text_query_gather`, `gather_rows`, `pixel_shuffle_rows` without
LN) are bit-exact gathers, checked bit for bit, above their grid caps.

Sine embedding, fp64.  The argument e = fl32(fl32(x * pre) / dim_t[d]) is two correctly rounded IEEE operations, so
the host reproduces it bit for bit: the product of two fp32 values is exact in fp64 and is rounded once; the fp64
quotient rounded to fp32 is the correctly rounded fp32 quotient (double rounding through a format of at least
2 * 24 + 2 bits is innocuous for division).  The library is built without fast-math, so sinf / cosf carry CUDA's
documented maximum error of 2 ulp: the fp32 output must lie within E = 2 ulp_fp32(z) of z = sin(e) / cos(e) in fp64
(err/E = 1 is 2 ulp).  The bf16 output must be RN_bf16 of the same call's fp32 output, bit for bit, and with the level
embedding RN_bf16(fl32(bf16(pos) + lvl)).

Detection top-k, exact.  The kernel's score is 1 / (1 + expf(-x)), torch.sigmoid's formula: scores must be
bit-equal to torch.sigmoid on the same GPU.  Against the true sigmoid in fp64 they hold |y - s| <= 2^-21 s + 2^-149
(expf within 2 ulp, two more roundings, subnormal steps of 2^-149), except where expf(-x) overflows (x < -88.72): there
fp32 gives exactly 0 while s < 2^-127, so y = 0 is accepted iff s <= 2^-127.  The oracle order is a stable sort of the
torch probabilities by (-p, flat index), NaN first (torch.topk ranks NaN above everything; among NaNs only the set is
checked); topk_indexes, box_idx, labels and boxes (the torch formula) must be identical to it.

Mask chain, fp64.  The source coordinate of an output index is one fp32 FMA, r = fma(dst + 0.5, scale, -0.5), with
scale = fl32(in / out), clamped at 0; i0 = (int)r, l1 = r - i0 (exact), l0 = fl32(1 - l1).  `mask_taps` reproduces
these in fp64 (the product is exact, then one rounding), and `mask_oracle` evaluates both bilinear stages in fp64 with
those weights.  The kernel evaluates each stage as l0 (l0' a + l1' b) + l1 (l0' c + l1' d): every one of the 16 terms
mu * lambda * m passes through at most 8 fp32 roundings (2 per nesting level, 4 levels), so its pre-threshold value
is within E = 8 * 2^-24 * sum_16 |mu lambda m| (+ 2^-126 for underflow) of the fp64 value.  fp32 sigmoid(v) > 0.5 is
decided as v > 0 once |v| >= 2^-20 (below that expf(-v) rounds so close to 1 that 1 / (1 + t) may round to 0.5), so
every pixel with |v64| > E + 2^-20 must equal v64 > 0; the rest are "undecided" and their fraction is reported.

Head stacking, exact: going to the stacks, rows tokens .. tokens_pad - 1 are +0 and the rest are the torch permute bit for
bit; coming back, NaN in the pad rows never reaches d(qkv); the packed pitch gap is neither read nor written.

Every output is a view into a larger sentinel-filled buffer (`Canvas`), prefilled with NaN or an impossible value:
every element inside must be written and every byte outside unchanged.  Regions a kernel must not read hold NaN or
point at NaN rows, always in bounds: a wrong kernel shows a wrong value, never a fault.  Every documented rejection
must return its code and leave every output buffer byte-identical.

`pytest -rP -s` prints the worst err/E per family (bf16_rounding.print_report) and the undecided mask-pixel fraction.
"""
import ctypes
import math
import random

import pytest
import torch

from visionllm_b200 import _lib
from bf16_rounding import REPORT, U, note_ratio, print_report, within

gpu = pytest.mark.gpu
OK, EINVAL, EUNSUPPORTED, EALIGN = 0, -1, -2, -3
NAN = float("nan")
SENTINEL = 4320.0                               # exact in bf16 / fp32; no output here equals it
EXTRA = {}                                      # family -> (undecided pixels, pixels) of the mask chain


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, (u, n) in sorted(EXTRA.items()):
        print(f"\n{k}: undecided pixels {u} / {n} = {u / max(n, 1):.2e}")
    EXTRA.clear()
    print_report("glue kernels")


# ---------------------------------------------------------------------------------------------------------------------
# helpers (device-agnostic; their CPU cases follow)
# ---------------------------------------------------------------------------------------------------------------------
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}


def bits(t):
    return t.view(_INT[t.dtype]) if t.dtype in _INT else t


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b.to(a.dtype)))


class Canvas:
    """An output of `shape` (row pitch `ld` >= shape[-1] for the last dimension, every outer dimension packed) inside a
    flat buffer of `fill`: 64 bytes (+ `shift` elements) before it, the pitch gaps, 64 bytes after.  The view is
    prefilled with `pre`.  `check(want)`: the view equals `want` bit for bit (or is only checked for being written
    when `want` is None) and every byte outside is unchanged; `untouched()`: no byte of the buffer changed."""

    def __init__(self, shape, dtype, ld=None, pre=NAN, fill=SENTINEL, shift=0, device="cuda"):
        shape = tuple(int(s) for s in shape)
        cols = shape[-1]
        rows = math.prod(shape[:-1])
        ld = cols if ld is None else int(ld)
        esz = torch.tensor([], dtype=dtype).element_size()
        lead = 64 // esz + shift
        self.buf = torch.full((lead + rows * ld + 64 // esz,), fill, dtype=dtype, device=device)
        strides = [1] * len(shape)
        if len(shape) >= 2:
            strides[-2] = ld
            for i in range(len(shape) - 3, -1, -1):
                strides[i] = strides[i + 1] * shape[i + 1]
        self.view = self.buf.as_strided(shape, strides, lead)
        self.view.fill_(pre)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=device)
        self.inside.as_strided(shape, strides, lead).fill_(True)
        self.before = bits(self.buf).clone()

    @property
    def ptr(self):
        return self.view.data_ptr()

    def check_outside(self, what):
        changed = (bits(self.buf) != self.before) & ~self.inside
        assert not bool(changed.any()), f"{what}: {int(changed.sum())} elements outside the output changed"

    def check(self, want, what):
        self.check_outside(what)
        diff = bits(self.view) != bits(want.to(self.view.device, self.view.dtype))
        if bool(diff.any()):
            i = tuple(diff.nonzero()[0].tolist())
            raise AssertionError(f"{what}: {int(diff.sum())} / {diff.numel()} elements differ, first at {i}: "
                                 f"got {self.view[i].item()!r}, want {want[i].item()!r}")

    def untouched(self, what):
        assert torch.equal(bits(self.buf), self.before), f"{what}: a rejected call wrote its output"


# ---- sequence assembly ----------------------------------------------------------------------------------------------
IMP, EMB, NE = 900, 910, 4
DET, SEG, GRD, POSE = 901, 902, 904, 903
TOOLS = [(DET, 0), (SEG, 0), (GRD, 0), (POSE, 1)]                  # (id, table): 0 emb_embeddings_det, 1 _pose
TOOLS8 = TOOLS + [(920, 1), (921, 0), (922, 1), (923, 0)]
TOOLS9 = TOOLS8 + [(924, 0)]


def make_ids(B, L, seed, tiles, tpt, tools=TOOLS, runs=3, imp_start=None):
    """input_ids [B, L]: random text tokens, one <im_patch> run of tiles[b] * tpt slots per sample (at imp_start[b] or
    at random), then up to `runs` tool tokens per sample each followed by NE pre-placed [EMB] slots."""
    g = random.Random(seed)
    ids = torch.randint(0, 800, (B, L), generator=torch.Generator().manual_seed(seed)).tolist()
    used = [[False] * L for _ in range(B)]
    for b in range(B):
        n = tiles[b] * tpt
        if n:
            s = imp_start[b] if imp_start else g.randrange(L - n + 1)
            for p in range(s, s + n):
                ids[b][p], used[b][p] = IMP, True
    for b in range(B):
        for _ in range(runs):
            if L <= NE:
                break
            p = g.randrange(L - NE)
            if any(used[b][p:p + NE + 1]):
                continue
            ids[b][p] = g.choice(tools)[0]
            for j in range(NE):
                ids[b][p + 1 + j] = EMB + (g.randrange(NE) if g.random() < 0.3 else 0)
            for q in range(p, p + NE + 1):
                used[b][q] = True
    return torch.tensor(ids, dtype=torch.int64)


def seq_oracle(ids, tools, tile_count, tpt, imp=IMP, emb=EMB, ne=NE):
    """Python-loop restatement of vllm_seq_index: (new_ids, kind, row, emb_pos lists, status).  A tool token whose
    slots leave the row or do not hold [EMB] ids sets status 1 and its slots are written up to the first bad one; a
    slot count that differs from the tile rows sets status 2, and slot k takes tile row k while there is one."""
    ids = ids.tolist()
    B, L = len(ids), len(ids[0])
    new = [r[:] for r in ids]
    kind = [[0] * L for _ in range(B)]
    row = [r[:] for r in ids]
    status = 0
    for tbl in (0, 1):                                              # det-class tools first, then pose (mv2.py:447-486)
        tset = {t for t, tb in tools if tb == tbl}
        for b in range(B):
            for p in range(L):
                if ids[b][p] not in tset:
                    continue
                for j in range(ne):
                    q = p + 1 + j
                    if q >= L or not emb <= ids[b][q] < emb + ne:
                        status |= 1
                        break
                    new[b][q], kind[b][q], row[b][q] = emb + j, 1 + tbl, j
    if imp >= 0 and tile_count is not None:
        start, starts = 0, []
        for c in tile_count:
            starts.append(start)
            start += c
        has = [imp in r for r in new]
        feat = [starts[b] * tpt + t for b in range(B) if has[b] for t in range(tile_count[b] * tpt)]
        slots = [(b, p) for b in range(B) for p in range(L) if new[b][p] == imp]
        if len(slots) != len(feat):
            status |= 2
        for (b, p), r in zip(slots, feat):
            kind[b][p], row[b][p] = 3, r
    emb_pos = [[p for p in range(L) if emb <= new[b][p] < emb + ne] for b in range(B)]
    return (torch.tensor(new, dtype=torch.int64), torch.tensor(kind, dtype=torch.uint8), torch.tensor(row, dtype=torch.int32),
            emb_pos, status)


def assemble_oracle(kind, row, embed, det, pose, image, base=None):
    """inputs_embeds[i] = the kind's source row: 0 embed[row] (or base[i]), 1 det[row], 2 pose[row], 3 image[row]."""
    kind, row = kind.long().reshape(-1), row.long().reshape(-1)
    out = torch.empty((kind.numel(), det.shape[1]), dtype=det.dtype, device=det.device)
    for k, src in enumerate((embed, det, pose, image)):
        sel = kind == k
        if k == 0 and base is not None:
            out[sel] = base.reshape(-1, det.shape[1])[sel]
        elif bool(sel.any()):
            out[sel] = src[row[sel]]
    return out


def text_query_oracle(hidden, emb_pos, ne, mx):
    """mv2.py:776-787: the first floor(count / ne) * ne [EMB] rows of each sample, zero padded to mx * ne rows."""
    B, L, C = hidden.shape
    tq = torch.zeros((B, mx * ne, C), dtype=hidden.dtype, device=hidden.device)
    tm = torch.zeros((B, mx), dtype=torch.uint8, device=hidden.device)
    for b in range(B):
        usable = len(emb_pos[b]) // ne * ne
        if usable:
            tq[b, :usable] = hidden[b, torch.tensor(emb_pos[b][:usable], device=hidden.device)]
            tm[b, :usable // ne] = 1
    return tq.view(B, mx, ne, C), tm


def pixel_shuffle_oracle(x, gw, gh, order):
    """x [tiles, gw * gh, C] -> [tiles * gw/2 * gh/2, 4C]: row (t, a, b) = the four tokens (2a + dy, 2b + dx) of the
    gw x gh token grid, (dy, dx) = (0,0), (0,1), (1,0), (1,1) for order 0 (mv2.py:381-392), (0,0), (1,0), (0,1), (1,1)
    for order 1 (HF SwinPatchMerging)."""
    tiles, _, C = x.shape
    x4 = x.reshape(tiles, gw, gh, C)
    chunks = ((0, 0), (0, 1), (1, 0), (1, 1)) if order == 0 else ((0, 0), (1, 0), (0, 1), (1, 1))
    return torch.cat([x4[:, dy::2, dx::2] for dy, dx in chunks], -1).reshape(-1, 4 * C)


# ---- sine embedding -------------------------------------------------------------------------------------------------
def f32(v):
    """The fp32 value of a python float (what ctypes passes for a `float` argument)."""
    return torch.tensor(v, dtype=torch.float32).item()


def sine_arg(x, pre, dim_t):
    """e = fl32(fl32(x * pre) / dim_t[d]) [rows, nd] fp32 from fp64 arithmetic: x * pre is exact in fp64 and rounded
    once; the fp64 quotient rounded to fp32 is the correctly rounded fp32 quotient."""
    x64 = x.double()
    if pre != 0.0:
        x64 = (x64 * f32(pre)).float().double()
    return (x64[:, None] / dim_t.double()[None, :]).float()


def sine_ref(e):
    """fp64 sin(e) at even d, cos(e) at odd d."""
    e64 = e.double()
    even = (torch.arange(e.shape[1], device=e.device) % 2 == 0)[None, :]
    return torch.where(even, torch.sin(e64), torch.cos(e64))


def ulp32(z):
    """ulp of fp32 at |z| (float64): 2^(e - 24) for |z| in [2^(e-1), 2^e), never below the subnormal step 2^-149."""
    _, e = torch.frexp(z.abs())
    q = (((e - 24).clamp(min=-149).to(torch.int64) + 1023) << 52).view(torch.float64)
    return torch.where(z == 0, torch.full_like(q, 2.0 ** -149), q)


# ---- detection top-k -------------------------------------------------------------------------------------------------
def topk_oracle(probs, k):
    """probs [B, n] -> flat indices [B, k]: stable sort by (-p, index), NaN above everything."""
    key = bits(probs.float()).long()                               # p >= 0: integer order == float order
    key = torch.where(probs.isnan(), torch.full_like(key, 1 << 40), key)
    return torch.sort(-key, dim=1, stable=True).indices[:, :k]


def box_oracle(pred_boxes, sizes_hw):
    """The torch formula of eval_det.py: cxcywh -> xyxy (util/box_ops.py:16-22), then * (w, h, w, h)."""
    cx, cy, w, h = pred_boxes.unbind(-1)
    xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)
    hh, ww = sizes_hw[:, 0], sizes_hw[:, 1]
    return xyxy * torch.stack([ww, hh, ww, hh], dim=1)[:, None, :]


def sigmoid_ok(y, x):
    """The fp64 bound of the module docstring: |y - s| <= 2^-21 s + 2^-149, or y == 0 where s <= 2^-127 (expf(-x)
    overflows).  Returns (ok mask, err / E)."""
    s = torch.sigmoid(x.double())
    E = 2.0 ** -21 * s + 2.0 ** -149
    err = (y.double() - s).abs()
    ok = (err <= E) | ((y == 0) & (s <= 2.0 ** -127))
    return ok, torch.where(y == 0, torch.zeros_like(err), err / E)


# ---- mask chain -----------------------------------------------------------------------------------------------------
def mask_scale(n_in, n_out):
    """fl32(n_in / n_out): ATen's (float)in / out, and the kernel's."""
    return f32(n_in / n_out)


def mask_taps(scale, n_out, n_in, device="cpu"):
    """(i0, i1, l0, l1) of every output index, float64 weights equal to the kernel's fp32 ones:
    r = fl32((dst + 0.5) * scale - 0.5) (one FMA) clamped at 0, i0 = (int)r, i1 = i0 + (i0 < n_in - 1),
    l1 = r - i0 (exact), l0 = fl32(1 - l1)."""
    dst = torch.arange(n_out, dtype=torch.float64, device=device)
    r = ((dst + 0.5) * scale - 0.5).float().double().clamp(min=0.0)
    i0 = r.floor()
    l1 = r - i0
    l0 = (1.0 - l1).float().double()
    i0 = i0.long()
    i1 = i0 + (i0 < n_in - 1).long()
    return i0, i1, l0, l1


def interp_matrix(scale, n_out, n_in, device="cpu"):
    """[n_out, n_in] float64: row o holds l0 at i0 and l1 at i1 (summed when they coincide)."""
    i0, i1, l0, l1 = mask_taps(scale, n_out, n_in, device)
    M = torch.zeros((n_out, n_in), dtype=torch.float64, device=device)
    o = torch.arange(n_out, device=device)
    M.index_put_((o, i0), l0, accumulate=True)
    M.index_put_((o, i1), l1, accumulate=True)
    return M


def mask_oracle(m, H, W, stride, ch, cw, oh, ow):
    """m [n, H, W] (fp32 values) -> (v64, E) [n, oh, ow]: both bilinear stages in float64 with the kernel's exact taps
    and weights; E = 8 u sum_16 |mu lambda m| + 2^-126."""
    ch, cw = min(ch, H * stride), min(cw, W * stride)
    dev = m.device
    Ay = interp_matrix(mask_scale(H, H * stride), H * stride, H, dev)[:ch]          # crop = the first ch / cw rows
    Ax = interp_matrix(mask_scale(W, W * stride), W * stride, W, dev)[:cw]
    By = interp_matrix(mask_scale(ch, oh), oh, ch, dev)
    Bx = interp_matrix(mask_scale(cw, ow), ow, cw, dev)
    Ty, Tx = By @ Ay, Bx @ Ax                                                       # composed, non-negative weights
    md = m.double()
    v = Ty @ md @ Tx.T
    E = 8 * U * (Ty @ md.abs() @ Tx.T) + 2.0 ** -126
    return v, E


def mask_decided(v, E):
    """Pixels whose sign the kernel must get right: |v64| > E + 2^-20."""
    return v.abs() > E + 2.0 ** -20


# ---------------------------------------------------------------------------------------------------------------------
# CPU cases of the helpers
# ---------------------------------------------------------------------------------------------------------------------
def _cpu_model():
    import torch.nn as nn
    from types import SimpleNamespace
    from visionllm_b200.modeling import B200VisionLLMv2Model

    class FakeViT(nn.Module):
        def __init__(self):
            super().__init__()
            self.config = SimpleNamespace(hidden_size=16, patch_size=2)

    class FakeLLM(nn.Module):
        def __init__(self):
            super().__init__()
            self.config = SimpleNamespace(hidden_size=16, vocab_size=1000)
            self.emb = nn.Embedding(1000, 16)

        @property
        def dtype(self):
            return self.emb.weight.dtype

        def get_input_embeddings(self):
            return self.emb

    cfg = SimpleNamespace(use_pixelshuffle=False, vl_bridge_type="linear", vis_output_layer=-1, num_embs=NE,
                          imp_token_id=IMP, emb_token_id=EMB, det_tool_id=DET, seg_tool_id=SEG, grd_tool_id=GRD,
                          pose_tool_id=POSE)
    return B200VisionLLMv2Model(cfg, FakeViT(), FakeLLM()).eval()


def test_seq_oracle_equals_the_model_indexing_and_the_reference_loop():
    from test_modeling_cpu import ref_emb_overwrite
    m = _cpu_model()
    for seed, (B, L, tiles, tpt) in enumerate([(4, 96, [2, 0, 1, 3], 8), (3, 200, [0, 2, 1], 16), (2, 40, [1, 1], 4)]):
        ids = make_ids(B, L, seed, tiles, tpt)
        tile_count = [t if t else 1 for t in tiles]                   # an image-less sample still owns a tile
        new, kind, row, emb_pos, status = seq_oracle(ids, TOOLS, tile_count, tpt)
        assert status == 0
        assert torch.equal(new, ref_emb_overwrite(ids, [t for t, _ in TOOLS], EMB, NE))
        with torch.no_grad():
            emb0 = m.llm.get_input_embeddings()(ids)
            ref_ids, ref_emb = m.inject_emb(ids, emb0)
            feats = torch.randn(sum(tile_count), tpt, 16)
            ref_emb = m.scatter_image_tokens(ref_ids, ref_emb, feats, tile_count)
            got = assemble_oracle(kind, row, m.llm.emb.weight, m.emb_embeddings_det.weight, m.emb_embeddings_pose.weight,
                                  feats.reshape(-1, 16))
            assert torch.equal(new, ref_ids) and torch.equal(got.view(B, L, 16), ref_emb)
            hidden = torch.randn(B, L, 16)
            tq_ref, tm_ref = m.gather_text_query(ref_ids, hidden)
            tq, tm = text_query_oracle(hidden, emb_pos, NE, tq_ref.shape[1])
            assert torch.equal(tq, tq_ref) and torch.equal(tm.bool(), tm_ref)
            base = torch.randn(B, L, 16)
            _, r_emb = m.inject_emb(ids, base)
            r_emb = m.scatter_image_tokens(ref_ids, r_emb, feats, tile_count)
            got = assemble_oracle(kind, row, None, m.emb_embeddings_det.weight, m.emb_embeddings_pose.weight,
                                  feats.reshape(-1, 16), base=base)
            assert torch.equal(got.view(B, L, 16), r_emb)


def test_seq_oracle_flags_and_edges():
    ids = torch.full((2, 8), 5, dtype=torch.int64)
    ids[0, 7] = DET                                                   # tool token in the last column
    assert seq_oracle(ids, TOOLS, None, 1)[4] == 1
    ids[0, 7] = 5
    ids[1, 5], ids[1, 6], ids[1, 7] = POSE, EMB, EMB                   # slots run past the row end: 2 of 4 written
    new, kind, row, _, st = seq_oracle(ids, TOOLS, None, 1)
    assert st == 1 and new[1, 6:].tolist() == [EMB, EMB + 1] and kind[1, 6:].tolist() == [2, 2] and row[1, 6:].tolist() == [0, 1]
    ids = torch.full((3, 6), 5, dtype=torch.int64)
    ids[0, :4] = IMP
    ids[2, 1:3] = IMP
    _, kind, row, _, st = seq_oracle(ids, TOOLS, [2, 5, 1], 2)        # 6 slots, tile rows 4 (sample 0) + 2 (sample 2)
    assert st == 0 and row[0, :4].tolist() == [0, 1, 2, 3] and row[2, 1:3].tolist() == [14, 15]
    _, kind, row, _, st = seq_oracle(ids, TOOLS, [1, 5, 1], 2)        # 6 slots, 4 tile rows: the last two keep kind 0
    assert st == 2 and row[0, :4].tolist() == [0, 1, 12, 13]
    assert kind[2, 1:3].tolist() == [0, 0] and row[2, 1:3].tolist() == [IMP, IMP]


def test_pixel_shuffle_oracle_is_the_reference_permutes():
    from visionllm_b200.modeling import pixel_shuffle
    x = torch.arange(2 * 4 * 6 * 8, dtype=torch.float32).view(2, 24, 8)
    ref = pixel_shuffle(x.view(2, 4, 6, 8), 0.5).reshape(-1, 32)
    assert torch.equal(pixel_shuffle_oracle(x, 4, 6, 0), ref)
    x4 = x.view(2, 4, 6, 8)
    swin = torch.cat([x4[:, 0::2, 0::2], x4[:, 1::2, 0::2], x4[:, 0::2, 1::2], x4[:, 1::2, 1::2]], -1).reshape(-1, 32)
    assert torch.equal(pixel_shuffle_oracle(x, 4, 6, 1), swin)


def test_sine_argument_reproduces_the_fp32_chain():
    import numpy as np
    g = torch.Generator().manual_seed(5)
    d = torch.arange(128, dtype=torch.float32)
    dim_t = 10000 ** (2 * torch.div(d, 2, rounding_mode="floor") / 128)
    for x, pre in ((torch.rand(4000, generator=g), 2 * math.pi), (torch.rand(4000, generator=g) * 7, 0.0),
                   ((torch.rand(4000, generator=g) - 0.5) * 2e4, 0.0), (torch.randn(4000, generator=g) * 1e3, 2 * math.pi)):
        want = ((x * torch.tensor(pre, dtype=torch.float32)) if pre else x)[:, None] / dim_t
        assert same_bits(sine_arg(x, pre, dim_t), want)
        xn = x.numpy()
        if pre:
            xn = xn * np.float32(pre)
        assert np.array_equal((xn[:, None] / dim_t.numpy()[None, :]).view(np.int32), sine_arg(x, pre, dim_t).numpy().view(np.int32))
    e = torch.tensor([[0.0, 0.0, 1.0, 1.0, 1e4, 1e4]], dtype=torch.float32)
    z = sine_ref(e)
    assert z[0, 0] == 0 and z[0, 1] == 1 and z[0, 2] == math.sin(1.0) and z[0, 5] == math.cos(1e4)
    assert ulp32(torch.tensor([1.0, 1.5, 0.75, 0.0, 2.0 ** -130], dtype=torch.float64)).tolist() == \
        [2.0 ** -23, 2.0 ** -23, 2.0 ** -24, 2.0 ** -149, 2.0 ** -149]


def test_topk_and_sigmoid_oracles():
    p = torch.tensor([[0.5, 0.7, NAN, 0.7, 0.0, 1.0, 0.5, NAN]])
    assert topk_oracle(p, 8).tolist() == [[2, 7, 5, 1, 3, 0, 6, 4]]
    x = torch.tensor([-120.0, -100.0, -88.0, -20.0, 0.0, 3.0, 17.0, float("-inf")])
    y = 1.0 / (1.0 + torch.exp(-x))                                 # the fp32 formula on the CPU
    ok, _ = sigmoid_ok(y, x)
    assert bool(ok.all()) and y[0] == 0 and y[1] == 0 and y[6] == 1.0
    bad = y.clone()
    bad[2] = 0.0                                                      # s(-88) = 6e-39 > 2^-127: must not be 0
    assert not bool(sigmoid_ok(bad, x)[0][2])
    b = torch.tensor([[[0.5, 0.25, 0.5, 0.25]]])
    assert box_oracle(b, torch.tensor([[100.0, 200.0]])).tolist() == [[[50.0, 12.5, 150.0, 37.5]]]


@pytest.mark.parametrize("H,W,stride,isz,tsz", [(16, 24, 4, (50, 96), (97, 61)), (8, 8, 2, (16, 16), (16, 16)),
                                                (12, 10, 4, (48, 33), (100, 70))])
def test_mask_oracle_equals_interpolate_in_float64(H, W, stride, isz, tsz):
    import torch.nn.functional as F
    m = torch.randn(3, H, W, generator=torch.Generator().manual_seed(H + W)) * 4
    v, E = mask_oracle(m, H, W, stride, isz[0], isz[1], tsz[0], tsz[1])
    up = F.interpolate(m.double()[:, None], size=(H * stride, W * stride), mode="bilinear", align_corners=False)
    ref = F.interpolate(up[:, :, :isz[0], :isz[1]], size=tsz, mode="bilinear", align_corners=False)[:, 0]
    # the oracle's weights are the fp32 ones, interpolate's the fp64 ones: they differ by an fp32 rounding of the tap
    # coordinate, far inside E's scale
    assert (v - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    assert bool((E > 0).all()) and float(E.max()) < 1e-4
    # the taps: in range, fp32 weights summing to 1 within one rounding, the coordinate within one fp32 rounding of
    # ATen's float64 one
    s = mask_scale(isz[1], tsz[1])
    i0, i1, l0, l1 = mask_taps(s, tsz[1], isz[1])
    assert bool(((0 <= i0) & (i0 <= i1) & (i1 < isz[1])).all()) and bool(((0 <= l1) & (l1 < 1)).all())
    assert torch.equal(l0.float().double(), l0) and torch.equal(l1.float().double(), l1)
    assert float((l0 + l1 - 1).abs().max()) <= 2.0 ** -24
    r64 = ((torch.arange(tsz[1], dtype=torch.float64) + 0.5) * s - 0.5).clamp(min=0)
    assert float(((i0 + l1) - r64).abs().max()) <= 2.0 ** -24 * float(r64.max())


def test_canvas_catches_a_single_changed_byte():
    for dtype, pre in ((torch.bfloat16, NAN), (torch.uint8, 0xAB), (torch.int64, -7)):
        c = Canvas((3, 5, 7), dtype, ld=9, pre=pre, fill=SENTINEL if dtype.is_floating_point else 0x5A, shift=1, device="cpu")
        want = torch.ones((3, 5, 7), dtype=dtype)
        with pytest.raises(AssertionError, match="differ"):
            c.check(want, "nothing written")
        c.untouched("nothing written")
        c.view.copy_(want)
        c.check(want, "written")
        raw = c.buf.view(torch.uint8)
        for pos in (0, raw.numel() - 1, (64 // c.buf.element_size() + 1 + 7) * c.buf.element_size()):   # lead, tail, gap
            raw[pos] ^= 1
            with pytest.raises(AssertionError, match="outside"):
                c.check(want, "outside byte")
            raw[pos] ^= 1
        with pytest.raises(AssertionError, match="rejected"):
            c.untouched("after a write")


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def stream():
    return torch.cuda.current_stream().cuda_stream


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def seq_call(ids, tools, tile_count, tpt, imp=IMP, ne=NE, batch=None):
    """vllm_seq_index into Canvas outputs; returns (rc, new_ids, kind, row, emb_pos, emb_count, status) canvases."""
    B, L = ids.shape
    B = B if batch is None else batch
    out = (Canvas((B, L), torch.int64, pre=-77777, fill=0x5A5A5A5A), Canvas((B, L), torch.uint8, pre=0xAB, fill=0xEE),
           Canvas((B, L), torch.int32, pre=-7777, fill=0x5A5A5A5A), Canvas((B, L), torch.int32, pre=-7777, fill=0x5A5A5A5A),
           Canvas((B,), torch.int32, pre=-7777, fill=0x5A5A5A5A), Canvas((1,), torch.int32, pre=0, fill=0x5A5A5A5A))
    tid = (ctypes.c_int64 * max(1, len(tools)))(*[t for t, _ in tools])
    ttb = (ctypes.c_int * max(1, len(tools)))(*[k for _, k in tools])
    if tile_count is not None:
        starts = [sum(tile_count[:b]) for b in range(len(tile_count))]
        meta = torch.tensor([starts, tile_count], dtype=torch.int32, device="cuda")
        ts, tc = meta[0].data_ptr(), meta[1].data_ptr()
    else:
        ts = tc = None
    rc = _lib.lib().vllm_seq_index(ids.data_ptr(), B, L, ctypes.cast(tid, ctypes.c_void_p), ctypes.cast(ttb, ctypes.c_void_p),
                                   len(tools), EMB, ne, imp, ts, tc, tpt, *[c.ptr for c in out], stream())
    torch.cuda.synchronize()
    return (rc,) + out


def seq_check(ids, tools, tile_count, tpt, what, imp=IMP, want_status=0):
    rc, new_ids, kind, row, emb_pos, emb_count, status = seq_call(ids.cuda(), tools, tile_count, tpt, imp=imp)
    assert rc == OK, what
    new, k, r, pos, st = seq_oracle(ids, tools, tile_count, tpt, imp=imp)
    assert st == want_status, f"{what}: the oracle's status is {st}"
    B, L = ids.shape
    new_ids.check(new, f"{what} new_ids")
    kind.check(k, f"{what} kind")
    row.check(r, f"{what} row")
    emb_count.check(torch.tensor([len(p) for p in pos], dtype=torch.int32), f"{what} emb_count")
    status.check(torch.tensor([st], dtype=torch.int32), f"{what} status")
    emb_pos.check_outside(f"{what} emb_pos")
    got = emb_pos.view.cpu()
    for b in range(B):
        assert got[b, :len(pos[b])].tolist() == pos[b], f"{what}: emb_pos of row {b}"
    return new, k, r, pos


# ---------------------------------------------------------------------------------------------------------------------
# 1. sequence assembly: exact
# ---------------------------------------------------------------------------------------------------------------------
SEQ_CASES = {
    # name: (B, L, tiles per sample, tokens per tile, <im_patch> run starts or None = random)
    "1x1": (1, 1, [0], 1, None),
    "1x31": (1, 31, [1], 8, None),
    "1x1023": (1, 1023, [3], 64, [1000 - 192]),
    "1x1024": (1, 1024, [2], 32, [1024 - 64]),
    "1x1025": (1, 1025, [1], 25, [1000]),                           # the run ends on position 1024: the second chunk
    "31x33": (31, 33, [1 if b % 3 else 0 for b in range(31)], 2, None),   # L = 33 ends one lane into pass 5's second warp step
    "3x1200": (3, 1200, [3, 0, 2], 100, [900, 0, 600]),              # runs straddle flat 1024 and 3072, an image-less sample between
    "2x1200": (2, 1200, [2, 1], 256, [600, 100]),                   # the chat step's shape; runs straddle 1024 and 1536
    "8x1100": (8, 1100, [3, 0, 1, 2, 0, 0, 3, 1], 64, None),         # B L >= 8192: eight chunks
    "1024x8": (1024, 8, [b % 2 for b in range(1024)], 4, None),      # B = MAX_SAMPLES
}


@gpu
@pytest.mark.parametrize("name", list(SEQ_CASES))
def test_seq_index_is_the_oracle(name):
    B, L, tiles, tpt, starts = SEQ_CASES[name]
    ids = make_ids(B, L, len(name), tiles, tpt, imp_start=starts)
    tile_count = [t if t else (b % 3) for b, t in enumerate(tiles)]  # image-less samples own 0 .. 2 skipped tiles
    seq_check(ids, TOOLS, tile_count, tpt, name)
    seq_check(ids, TOOLS, None, tpt, name + " text-only")              # no tile arrays: every position keeps kind 0 / 1 / 2
    seq_check(ids, TOOLS, tile_count, tpt, name + " no imp id", imp=-1)


@gpu
def test_seq_index_eight_tools_det_and_pose_in_one_row():
    ids = make_ids(4, 200, 8, [1, 0, 2, 1], 16, tools=TOOLS8, runs=10)
    ids[0] = 5                                                        # row 0 rebuilt: no <im_patch>, hand-placed tools
    ids[0, 10:15] = torch.tensor([921, EMB, EMB + 1, EMB + 2, EMB + 3])
    ids[0, 150:160] = torch.tensor([DET, EMB, EMB, EMB, EMB, POSE, EMB, EMB + 3, EMB, EMB])   # det and pose back to back
    ids[0, 160:165] = torch.tensor([922, EMB, EMB, EMB, EMB])
    _, kind, _, _ = seq_check(ids, TOOLS8, [1, 2, 2, 1], 16, "eight tools")
    assert kind[0, 151:160].tolist() == [1, 1, 1, 1, 0, 2, 2, 2, 2] and kind[0, 161:165].tolist() == [2] * 4


@gpu
def test_seq_index_status_flags():
    ids = make_ids(2, 64, 3, [1, 1], 8, imp_start=[0, 0])
    ids[0, 63] = SEG                                                 # a tool token in the last column
    seq_check(ids, TOOLS, [1, 1], 8, "tool in the last column", want_status=1)
    ids[0, 63] = 7
    ids[1, 60:64] = torch.tensor([POSE, EMB, EMB, EMB])               # slots run past the row end
    seq_check(ids, TOOLS, [1, 1], 8, "slots past the row end", want_status=1)
    ids[1, 60] = 7
    ids[1, 20:25] = torch.tensor([DET, EMB, 5, EMB, EMB])             # insert form: a slot without an [EMB] id
    seq_check(ids, TOOLS, [1, 1], 8, "insert form", want_status=1)
    ids = make_ids(3, 1200, 4, [2, 0, 3], 100, imp_start=[950, 0, 300])
    seq_check(ids, TOOLS, [1, 1, 3], 100, "fewer tile rows than slots", want_status=2)
    seq_check(ids, TOOLS, [4, 1, 3], 100, "more tile rows than slots", want_status=2)


@gpu
def test_seq_index_rejections_leave_the_outputs_untouched():
    ids = make_ids(1025, 2, 1, [0] * 1025, 1).cuda()               # full-size inputs and outputs: a missed rejection is a value
    for B, tools, want in ((1025, TOOLS, EUNSUPPORTED), (4, TOOLS9, EINVAL)):
        rc, *outs = seq_call(ids, tools, None, 1, batch=B)
        assert rc == want, (B, len(tools), rc)
        for c in outs:
            c.untouched(f"B={B} tools={len(tools)}")
    rc, *outs = seq_call(ids[:4], TOOLS8, None, 1, ne=0)
    assert rc == EINVAL
    for c in outs:
        c.untouched("num_embs 0")
    rc, *_ = seq_call(ids[:1024], TOOLS8, None, 1)
    assert rc == OK


def _assemble_sources(rows, C, seed, V=1000, R=700):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kind = torch.randint(0, 4, (rows,), device="cuda", generator=g).to(torch.uint8)
    hi = torch.tensor([V, NE, NE, R], device="cuda")[kind.long()]
    row = (torch.rand(rows, device="cuda", generator=g) * hi).long().clamp(max=hi - 1).int()
    src = [torch.randn(n, C, device="cuda", generator=g).bfloat16() for n in (V, NE, NE, R)]
    base = torch.randn(rows, C, device="cuda", generator=g).bfloat16()
    return kind, row, src, base


@gpu
@pytest.mark.parametrize("rows,C", [(37, 64), (2500, 8), (2500, 64), (2200, 4096)])
def test_assemble_embeds_copies_every_row_bit_exact(rows, C):
    assert rows < 100 or rows > 16 * num_sms()                      # one pass, or the grid-stride loop
    kind, row, (embed, det, pose, image), base = _assemble_sources(rows, C, rows + C)
    for with_base in (False, True):
        out = Canvas((rows, C), torch.bfloat16)
        rc = _lib.lib().vllm_assemble_embeds_bf16(kind.data_ptr(), row.data_ptr(), None if with_base else embed.data_ptr(),
                                                  det.data_ptr(), pose.data_ptr(), image.data_ptr(),
                                                  base.data_ptr() if with_base else None, out.ptr, rows, C, stream())
        torch.cuda.synchronize()
        assert rc == OK
        out.check(assemble_oracle(kind, row, embed, det, pose, image, base if with_base else None), f"base={with_base}")
    out = Canvas((rows, C), torch.bfloat16)
    for C_bad, want in ((C + 4, EINVAL), (0, EINVAL)):
        rc = _lib.lib().vllm_assemble_embeds_bf16(kind.data_ptr(), row.data_ptr(), embed.data_ptr(), det.data_ptr(),
                                                  pose.data_ptr(), image.data_ptr(), None, out.ptr, rows, C_bad, stream())
        assert rc == want
    rc = _lib.lib().vllm_assemble_embeds_bf16(kind.data_ptr(), row.data_ptr(), None, det.data_ptr(), pose.data_ptr(),
                                              image.data_ptr(), None, out.ptr, rows, C, stream())
    assert rc == EINVAL                                               # neither the token table nor base_embeds
    torch.cuda.synchronize()
    out.untouched("assemble rejections")


@gpu
@pytest.mark.parametrize("B,L,C,ne,counts,mx", [(3, 64, 64, 4, [0, 7, 16], 6), (8, 400, 64, 4, None, 80),
                                                (2, 40, 4096, 4, [9, 12], 4), (5, 33, 8, 1, [0, 3, 32, 1, 5], 40)])
def test_text_query_gather_is_exact_and_zero_padded(B, L, C, ne, counts, mx):
    g = random.Random(B * L + C)
    if counts is None:
        counts = [g.randrange(0, 300) for _ in range(B)]
    emb_pos = [sorted(g.sample(range(L - 1), c)) for c in counts]        # position L - 1 is never an [EMB] slot
    hidden = torch.full((B, L, C), NAN, dtype=torch.bfloat16, device="cuda")   # rows no usable [EMB] names stay NaN
    for b in range(B):
        usable = counts[b] // ne * ne
        if usable:
            hidden[b, torch.tensor(emb_pos[b][:usable], device="cuda")] = torch.randn(usable, C, device="cuda").bfloat16()
    pos_t = torch.full((B, L), L - 1, dtype=torch.int32)                # entries past the count point at a NaN row
    for b in range(B):
        pos_t[b, :counts[b]] = torch.tensor(emb_pos[b], dtype=torch.int32)
    pos_t = pos_t.cuda()
    cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
    assert mx > max(counts) // ne
    if B == 8:
        assert B * mx * ne > 16 * num_sms()                          # the grid-stride loop
    tq, tm = Canvas((B, mx, ne, C), torch.bfloat16), Canvas((B, mx), torch.uint8, pre=0xAB, fill=0xEE)
    rc = _lib.lib().vllm_text_query_gather_bf16(hidden.data_ptr(), pos_t.data_ptr(), cnt.data_ptr(), B, L, C, ne, mx,
                                                tq.ptr, tm.ptr, stream())
    torch.cuda.synchronize()
    assert rc == OK
    want_tq, want_tm = text_query_oracle(hidden, emb_pos, ne, mx)
    tq.check(want_tq, "text_query")
    tm.check(want_tm, "text_query_masks")
    assert not bool(tq.view.isnan().any())
    tq2, tm2 = Canvas((B, mx, ne, C), torch.bfloat16), Canvas((B, mx), torch.uint8, pre=0xAB, fill=0xEE)
    for args in ((B, L, C + 4, ne, mx), (B, L, C, 0, mx), (B, L, C, ne, -1)):
        assert _lib.lib().vllm_text_query_gather_bf16(hidden.data_ptr(), pos_t.data_ptr(), cnt.data_ptr(), *args,
                                                      tq2.ptr, tm2.ptr, stream()) == EINVAL
    torch.cuda.synchronize()
    tq2.untouched("text_query rejections")
    tm2.untouched("text_query_masks rejections")


@gpu
@pytest.mark.parametrize("src_rows,C,n", [(50, 128, 6), (3000, 96, 100000), (777, 8, 5000), (40, 1016, 3000),
                                          (33, 1024, 3000), (9, 4096, 2500)])
def test_gather_rows_both_kernels_above_their_grid_caps(src_rows, C, n):
    g = torch.Generator(device="cuda").manual_seed(src_rows + C)
    ld = C + 24
    src = torch.full((src_rows, ld), NAN, dtype=torch.bfloat16, device="cuda")        # NaN pitch gap
    named = torch.randperm(src_rows, device="cuda", generator=g)[:max(1, src_rows * 3 // 4)]   # the rest stay NaN
    src[named, :C] = torch.randn(named.numel(), C, device="cuda", generator=g).bfloat16()
    if n == 6:
        idx = torch.tensor([0, src_rows - 1, 7, 7, -1, -src_rows], device="cuda")
        src[idx, :C] = torch.randn(6, C, device="cuda", generator=g).bfloat16()
    else:
        pick = named[torch.randint(0, named.numel(), (n,), device="cuda", generator=g)]
        neg = torch.rand(n, device="cuda", generator=g) < 0.4
        idx = torch.where(neg, pick - src_rows, pick)                    # python-style negative indices
    nvec = C // 8
    if n == 100000:
        assert nvec < 128 and n * nvec > 32 * 256 * num_sms()         # the flat kernel's grid-stride loop
    if nvec >= 128:
        assert n > 16 * num_sms()                                     # the row kernel's grid-stride loop
    dst = Canvas((n, C), torch.bfloat16)
    rc = _lib.lib().vllm_gather_rows_bf16(src.data_ptr(), ld, src_rows, idx.data_ptr(), n, C, dst.ptr, stream())
    torch.cuda.synchronize()
    assert rc == OK
    dst.check(src[:, :C][idx], "gather_rows")
    bad = Canvas((n, C), torch.bfloat16)
    for args, want in (((src.data_ptr(), C - 8, src_rows, idx.data_ptr(), n, C, bad.ptr), EINVAL),
                       ((src.data_ptr(), ld + 4, src_rows, idx.data_ptr(), n, C, bad.ptr), EALIGN),
                       ((src.data_ptr(), ld, src_rows, idx.data_ptr(), n, C, bad.ptr + 2), EALIGN),
                       ((src.data_ptr(), ld, src_rows, idx.data_ptr(), n, C + 4, bad.ptr), EINVAL)):
        assert _lib.lib().vllm_gather_rows_bf16(*args, stream()) == want
    torch.cuda.synchronize()
    bad.untouched("gather_rows rejections")


PS_CASES = [  # (tiles, grid rows, grid cols, C, skip tokens): C walks the VPT ladder 2 / 4 / 8 and its edges
    (3, 4, 4, 8, 1), (2, 2, 2, 1024, 1), (2, 4, 6, 1032, 0), (1, 6, 2, 2048, 3), (2, 2, 4, 2056, 1), (2, 4, 2, 4096, 1),
    (5, 16, 12, 64, 1),
]


@gpu
@pytest.mark.parametrize("tiles,gw,gh,C,skip", PS_CASES)
@pytest.mark.parametrize("order", [0, 1])
def test_pixel_shuffle_without_ln_is_an_exact_permutation(tiles, gw, gh, C, skip, order):
    g = torch.Generator(device="cuda").manual_seed(tiles * 1000 + C + order)
    T = skip + gw * gh
    ld_token = C + 16
    ld_tile = T * ld_token + 40
    buf = torch.full((tiles * ld_tile + 64,), NAN, dtype=torch.bfloat16, device="cuda")   # pitch gaps and CLS tokens NaN
    x = buf.as_strided((tiles, gw * gh, C), (ld_tile, ld_token, 1), skip * ld_token)
    x.copy_(torch.randn(tiles, gw * gh, C, device="cuda", generator=g).bfloat16())
    rows = tiles * (gw // 2) * (gh // 2)
    y = Canvas((rows, 4 * C), torch.bfloat16)
    rc = _lib.lib().vllm_pixel_shuffle_rows_bf16(buf.data_ptr(), ld_tile, ld_token, skip, tiles, gw, gh, C, None, None,
                                                 1e-5, y.ptr, order, stream())
    torch.cuda.synchronize()
    assert rc == OK
    y.check(pixel_shuffle_oracle(x.contiguous(), gw, gh, order), f"order {order}")


@gpu
def test_pixel_shuffle_rejections_leave_the_output_untouched():
    C, gw, gh = 4104, 2, 2                                           # 4C / 8 = 2052 vectors: past the VPT ladder
    x = torch.randn(1, 1 + gw * gh, C, device="cuda").bfloat16()
    y = Canvas((1, 4 * C), torch.bfloat16)
    L = _lib.lib()
    for args, want in (((x.data_ptr(), x.stride(0), C, 1, 1, gw, gh, C), EUNSUPPORTED),
                       ((x.data_ptr(), x.stride(0), 8, 1, 1, 3, 2, 8), EINVAL),
                       ((x.data_ptr(), x.stride(0), 8, 1, 1, 2, 2, 12), EINVAL),
                       ((x.data_ptr(), x.stride(0), 12, 1, 1, 2, 2, 8), EALIGN),
                       ((x.data_ptr() + 2, x.stride(0), 8, 1, 1, 2, 2, 8), EALIGN)):
        assert L.vllm_pixel_shuffle_rows_bf16(*args, None, None, 1e-5, y.ptr, 0, stream()) == want, args
    assert L.vllm_pixel_shuffle_rows_bf16(x.data_ptr(), x.stride(0), 8, 1, 1, 2, 2, 8, None, None, 1e-5, y.ptr, 2,
                                          stream()) == EINVAL
    torch.cuda.synchronize()
    y.untouched("pixel_shuffle rejections")


# ---------------------------------------------------------------------------------------------------------------------
# 2. sine embedding: fp64
# ---------------------------------------------------------------------------------------------------------------------
def _dim_t(nd, temperature=10000.0):
    d = torch.arange(nd, dtype=torch.float32, device="cuda")
    return temperature ** (2 * torch.div(d, 2, rounding_mode="floor") / nd)


def sine_run(feats_mat, cols, stride, pre, dim_t, rows, ldo, rpb=0, obs=0, nslab=1, add_row=None):
    """Runs fp32, bf16 and (if add_row) bf16 + add_row on the same inputs into Canvas outputs and checks the whole
    contract.  feats_mat: fp32 buffer holding feature f at feats_mat.view(-1)[cols[f] + r * stride]."""
    nf, nd = len(cols), dim_t.numel()
    W = nf * nd
    base = feats_mat.data_ptr()
    ptr = [base + 4 * c for c in cols] + [None] * (4 - nf)

    def out_canvas(dtype):
        if rpb:
            c = Canvas((nslab, obs), dtype)                        # slabs obs elements apart, rows ldo apart inside
            v = c.buf.as_strided((nslab, rpb, W), (obs, ldo, 1), c.view.storage_offset())
            c.inside.zero_()
            c.inside.as_strided((nslab, rpb, W), (obs, ldo, 1), c.view.storage_offset()).fill_(True)
            c.buf.fill_(SENTINEL)
            v.fill_(NAN)
            c.before = bits(c.buf).clone()
            c.view = v
            return c
        return Canvas((rows, W), dtype, ld=ldo)

    def call(c, bf16, add):
        rc = _lib.lib().vllm_sine_embed_f32(*ptr, stride, nf, f32(pre), dim_t.data_ptr(), nd, rows, c.ptr, ldo, int(bf16),
                                            rpb, obs, add, stream())
        torch.cuda.synchronize()
        assert rc == OK
        return c.view.reshape(rows, W)

    flat = feats_mat.reshape(-1)
    x = torch.stack([flat[c + stride * torch.arange(rows, device="cuda")] for c in cols])   # [nf, rows]
    e = torch.cat([sine_arg(x[f], pre, dim_t) for f in range(nf)], 1)
    z = sine_ref(e)
    o32 = out_canvas(torch.float32)
    y = call(o32, False, None)
    o32.check_outside("sine fp32")
    assert bool(y.isfinite().all()), "sine fp32: an output element is unwritten"
    within(y, z, 2 * ulp32(z), "sine fp32 (E = 2 ulp)", f"nf={nf} nd={nd} pre={pre}")
    o16 = out_canvas(torch.bfloat16)
    y16 = call(o16, True, None)
    o16.check_outside("sine bf16")
    assert same_bits(y16, y.bfloat16()), "sine bf16 != RN_bf16 of the fp32 output"
    if add_row is not None:
        oa = out_canvas(torch.bfloat16)
        ya = call(oa, True, add_row.data_ptr())
        oa.check_outside("sine bf16 + add_row")
        assert same_bits(ya, (y.bfloat16().float() + add_row.float()[None, :]).bfloat16()), "sine bf16 + add_row"
    return y


@gpu
@pytest.mark.parametrize("nd", [8, 16, 128])
@pytest.mark.parametrize("nf", [1, 2, 3, 4])
def test_sine_embed_within_two_ulp_of_fp64(nf, nd):
    g = torch.Generator(device="cuda").manual_seed(nf * 100 + nd)
    rows, S = 37, 2 * nf + 1                                         # features are columns 0, 2, .. of [rows, S]; the rest NaN
    mat = torch.full((rows, S), NAN, device="cuda")
    cols = [2 * f for f in range(nf)]
    for c in cols:
        mat[:, c] = torch.rand(rows, device="cuda", generator=g) * (1.0 + 3 * c)
    add = (torch.randn(nf * nd, device="cuda", generator=g) * 0.5).bfloat16()
    for pre in (0.0, 2 * math.pi):
        sine_run(mat, cols, S, pre, _dim_t(nd), rows, nf * nd + 8, add_row=add)


@gpu
def test_sine_embed_level_slabs_and_the_grid_stride_loop():
    g = torch.Generator(device="cuda").manual_seed(3)
    nd, nf = 128, 2
    dim_t = _dim_t(nd, 20.0)
    add = (torch.randn(nf * nd, device="cuda", generator=g) * 0.5).bfloat16()
    # one level of a [2, S, 256] buffer: two slabs of rpb rows with a gap between them
    rpb = 50
    mat = (torch.rand(2 * rpb, 2, device="cuda", generator=g) * 2 * math.pi).contiguous()
    sine_run(mat, [0, 1], 2, 0.0, dim_t, 2 * rpb, 256, rpb=rpb, obs=rpb * 256 + 24, nslab=2, add_row=add)
    # above the grid cap (16 CTAs x 256 threads per SM): 2 x 16,387 level-0 rows of two contiguous maps
    rpb = 16387
    assert 2 * rpb * nf * nd // 8 > 16 * 256 * num_sms()
    ye = torch.rand(2 * rpb, device="cuda", generator=g) * 2 * math.pi
    xe = torch.rand(2 * rpb, device="cuda", generator=g) * 2 * math.pi
    mat = torch.stack([ye, xe])                                       # feature f at f * rows + r
    sine_run(mat, [0, 2 * rpb], 1, 0.0, dim_t, 2 * rpb, 256, rpb=rpb, obs=rpb * 256 + 8, nslab=2, add_row=add)
    sine_run(mat, [0, 2 * rpb], 1, 2 * math.pi, dim_t, 2 * rpb, 264)


@gpu
def test_sine_embed_wide_arguments():
    g = torch.Generator(device="cuda").manual_seed(9)
    rows = 4096
    mat = ((torch.rand(rows, 1, device="cuda", generator=g) - 0.5) * 2e4).contiguous()
    dim_t = torch.tensor([1.0, 1.0, 1.5, 1.5, 3.0, 3.0, 7.0, 7.0], device="cuda")
    sine_run(mat, [0], 1, 0.0, dim_t, rows, 8)
    sine_run(mat, [0], 1, 2 * math.pi, dim_t, rows, 8)


@gpu
def test_sine_embed_rejections_leave_the_output_untouched():
    f = torch.rand(64, device="cuda")
    dim_t = _dim_t(16)
    o = Canvas((64, 64), torch.float32, ld=64)
    L = _lib.lib()
    p = f.data_ptr()
    for args, want in (((p, p, p, p, 1, 5, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 64, 0, 0, 0, None), EINVAL),   # nfeat 5
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 12, 64, o.ptr, 64, 0, 0, 0, None), EINVAL),  # nd % 8
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 24, 0, 0, 0, None), EINVAL),  # ldo < W
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 32, 0, 32, 1000, None), EINVAL),  # obs
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 32, 0, 0, 0, p), EINVAL),     # add_row, fp32
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 34, 0, 0, 0, None), EALIGN),
                       ((p, p, None, None, 1, 2, 0.0, dim_t.data_ptr(), 16, 32, o.ptr + 4, 32, 0, 0, 0, None), EALIGN),
                       ((p, p, None, None, 0, 2, 0.0, dim_t.data_ptr(), 16, 64, o.ptr, 32, 0, 0, 0, None), EINVAL)):
        assert L.vllm_sine_embed_f32(*args, stream()) == want, args
    torch.cuda.synchronize()
    o.untouched("sine rejections")


# ---------------------------------------------------------------------------------------------------------------------
# 3. detection top-k: exact
# ---------------------------------------------------------------------------------------------------------------------
def det_call(logits, ld, K, pred_boxes, sizes, k, B=None, boxes_shift=0, boxes_in_shift=0):
    """vllm_det_postprocess_f32 on logits [B, Q, ld] into Canvas outputs: (rc, scores, idx, box_idx, labels, boxes)."""
    B = logits.shape[0] if B is None else B
    Q = logits.shape[1]
    kc = max(k, 1)
    outs = (Canvas((B, kc), torch.float32, pre=-1.0), Canvas((B, kc), torch.int64, pre=-7, fill=0x5A5A5A5A),
            Canvas((B, kc), torch.int64, pre=-7, fill=0x5A5A5A5A), Canvas((B, kc), torch.int64, pre=-7, fill=0x5A5A5A5A),
            Canvas((B, kc, 4), torch.float32))
    rc = _lib.lib().vllm_det_postprocess_f32(logits.data_ptr(), pred_boxes.data_ptr() + boxes_in_shift, sizes.data_ptr(), B,
                                             Q, K, ld, k, *[c.ptr for c in outs[:4]], outs[4].ptr + boxes_shift, stream())
    torch.cuda.synchronize()
    return (rc,) + outs


def det_check(logits, K, pred_boxes, sizes, k, what):
    """The whole top-k contract for logits [B, Q, ld] (columns K .. ld hold NaN)."""
    B, Q, ld = logits.shape
    rc, scores, idx, box_idx, labels, boxes = det_call(logits, ld, K, pred_boxes, sizes, k)
    assert rc == OK, what
    for c in (scores, idx, box_idx, labels, boxes):
        c.check_outside(what)
    probs = torch.sigmoid(logits[:, :, :K]).reshape(B, Q * K)
    want = topk_oracle(probs, k)
    got = idx.view
    n_nan = probs.isnan().sum(1)
    for b in range(B):
        m = min(int(n_nan[b]), k)
        assert sorted(got[b, :m].tolist()) == sorted(want[b, :m].tolist()), f"{what}: image {b}: the NaN set"
        assert torch.equal(got[b, m:], want[b, m:]), \
            f"{what}: image {b}: order differs at {int((got[b, m:] != want[b, m:]).nonzero()[0]) + m}"
    # every output follows the kernel's own indices (the NaN block may be in any order)
    s = probs.gather(1, got)
    nan = s.isnan()
    assert torch.equal(scores.view.isnan(), nan) and same_bits(scores.view[~nan], s[~nan]), f"{what}: scores != torch.sigmoid"
    x = logits[:, :, :K].reshape(B, Q * K).gather(1, got)
    ok, ratio = sigmoid_ok(scores.view[~nan], x[~nan])
    assert bool(ok.all()), f"{what}: a score outside the fp64 bound of the sigmoid"
    note_ratio("det scores vs fp64 sigmoid", float(ratio.max()) if ratio.numel() else 0.0)
    assert torch.equal(box_idx.view, got // K) and torch.equal(labels.view, got % K), what
    want_boxes = box_oracle(pred_boxes, sizes).gather(1, (got // K)[:, :, None].expand(B, k, 4))
    assert same_bits(boxes.view, want_boxes), f"{what}: boxes != the torch formula"
    return scores.view, got, boxes.view


def _det_inputs(B, Q, K, ld, seed, gen):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.full((B, Q, ld), NAN, device="cuda")               # the ld gap is NaN: never read
    logits[:, :, :K] = gen(g, (B, Q, K))
    pred_boxes = torch.rand(B, Q, 4, device="cuda", generator=g)
    sizes = torch.tensor([[480.0, 640.0], [1024.0, 1024.0], [333.0, 500.0]][:B], device="cuda")
    return logits, pred_boxes, sizes


def _quantised(g, shape):
    return torch.round(torch.randn(shape, device="cuda", generator=g) * 4) / 4      # ~60 distinct values: heavy ties


def _saturated(g, shape):
    x = torch.randn(shape, device="cuda", generator=g) * 3
    hot = torch.rand(shape, device="cuda", generator=g) < 0.02
    return torch.where(hot, 17 + torch.rand(shape, device="cuda", generator=g) * 10, x)   # prob 1.0 in ~2 % of slots


def _underflow(g, shape):
    x = torch.round((-88 - torch.rand(shape, device="cuda", generator=g) * 16) * 4) / 4      # subnormal and 0 probabilities
    pad = torch.rand(shape, device="cuda", generator=g) < 0.1
    return torch.where(pad, torch.full_like(x, float("-inf")), x)                           # -inf class padding


def _with_nan(g, shape):
    x = torch.randn(shape, device="cuda", generator=g) * 3
    x.view(-1)[torch.randperm(x.numel(), device="cuda", generator=g)[:37]] = NAN
    return x


DET_CASES = {   # name: (B, Q, K, ld, logits, k values)
    "ties 900x256": (2, 900, 256, 264, _quantised, (1, 2, 1023, 1024)),
    "saturated": (2, 900, 16, 16, _saturated, (1024, 1000)),
    "underflow": (1, 64, 16, 20, _underflow, (1024, 1000, 7)),
    "k = n 21": (2, 7, 3, 8, _quantised, (21,)),
    "nan": (3, 300, 80, 84, _with_nan, (100, 37, 1024)),
}


@gpu
@pytest.mark.parametrize("name", list(DET_CASES))
def test_det_topk_is_the_stable_sort(name):
    B, Q, K, ld, gen, ks = DET_CASES[name]
    logits, pred_boxes, sizes = _det_inputs(B, Q, K, ld, len(name), gen)
    for k in ks:
        det_check(logits, K, pred_boxes, sizes, k, f"{name} k={k}")


@gpu
def test_det_topk_image_of_a_batch_equals_the_image_alone():
    logits, pred_boxes, sizes = _det_inputs(3, 900, 256, 256, 77, _quantised)
    _, full_s, full_i, full_b, full_l, full_x = det_call(logits, 256, 256, pred_boxes, sizes, 1024)
    for b in range(3):
        _, s, i, bi, lb, x = det_call(logits[b:b + 1], 256, 256, pred_boxes[b:b + 1], sizes[b:b + 1], 1024)
        for a, c in ((full_s, s), (full_i, i), (full_b, bi), (full_l, lb), (full_x, x)):
            assert same_bits(a.view[b:b + 1], c.view), f"image {b}"


@gpu
def test_det_topk_k_equals_n_1024():
    logits, pred_boxes, sizes = _det_inputs(2, 32, 32, 40, 5, _quantised)
    det_check(logits, 32, pred_boxes, sizes, 1024, "k = n = 1024")


@gpu
def test_det_topk_rejections_leave_the_outputs_untouched():
    logits, pred_boxes, sizes = _det_inputs(1, 64, 32, 40, 6, _quantised)
    pb = torch.zeros(1, 65, 4, device="cuda")                         # one row of slack for the shifted pointer
    pb[:, :64] = pred_boxes
    for args, want in (((40, 32, 1025), EUNSUPPORTED), ((40, 32, 64 * 32 + 1), EUNSUPPORTED), ((20, 32, 16), EINVAL),
                       ((40, 32, 0), EINVAL)):
        ld, K, k = args
        rc, *outs = det_call(logits, ld, K, pb, sizes, k)
        assert rc == want, args
        for c in outs:
            c.untouched(f"det {args}")
    for kw in ({"boxes_shift": 4}, {"boxes_in_shift": 4}):
        rc, *outs = det_call(logits, 40, 32, pb, sizes, 16, **kw)
        assert rc == EALIGN, kw
        for c in outs:
            c.untouched(f"det {kw}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. mask chain: fp64
# ---------------------------------------------------------------------------------------------------------------------
def mask_call(masks, box_idx, stride, crop, out_hw, shift=0, out=None):
    """vllm_mask_postprocess_f32 of one image into a uint8 Canvas (base `shift` bytes past 16-byte alignment)."""
    Q, H, W = masks.shape
    n = box_idx.numel()
    if out is None:
        out = Canvas((n, out_hw[0], out_hw[1]), torch.uint8, pre=0xCD, fill=0xEE, shift=shift)
    rc = _lib.lib().vllm_mask_postprocess_f32(masks.data_ptr(), box_idx.data_ptr(), n, H, W, stride, crop[0], crop[1],
                                              out_hw[0], out_hw[1], out.ptr, stream())
    torch.cuda.synchronize()
    return rc, out


def mask_check(masks, box_idx, stride, crop, out_hw, what, shift=0):
    Q, H, W = masks.shape
    rc, out = mask_call(masks, box_idx, stride, crop, out_hw, shift)
    assert rc == OK, what
    out.check_outside(what)
    got = out.view
    assert bool((got <= 1).all()), f"{what}: a byte outside {{0, 1}} (unwritten: 0xCD)"
    v, E = mask_oracle(masks[box_idx], H, W, stride, crop[0], crop[1], out_hw[0], out_hw[1])
    dec = mask_decided(v, E)
    wrong = dec & (got.bool() != (v > 0))
    assert not bool(wrong.any()), f"{what}: {int(wrong.sum())} decided pixels wrong, first at {tuple(wrong.nonzero()[0].tolist())}"
    u, n = EXTRA.get("mask chain", (0, 0))
    EXTRA["mask chain"] = (u + int((~dec).sum()), n + dec.numel())
    return got


MASK_CASES = [(64, 64, 4, (250, 256), (480, 517)), (32, 40, 4, (128, 160), (128, 160)),
              (56, 56, 4, (200, 224), (1000, 1333)), (16, 24, 2, (31, 47), (97, 61))]


@gpu
@pytest.mark.parametrize("H,W,stride,crop,out_hw", MASK_CASES)
def test_mask_chain_decides_every_pixel_the_fp64_value_decides(H, W, stride, crop, out_hw):
    g = torch.Generator(device="cuda").manual_seed(H * 7 + W)
    masks = torch.randn(20, H, W, device="cuda", generator=g) * 4
    bi = torch.randint(0, 20, (9,), device="cuda", generator=g)
    got = mask_check(masks, bi, stride, crop, out_hw, f"{H}x{W}")
    for d in (0, 4, 8):                                              # each detection alone: the same bytes
        _, alone = mask_call(masks, bi[d:d + 1], stride, crop, out_hw)
        assert torch.equal(alone.view[0], got[d]), f"detection {d} alone"
    # a crop past mask * stride is clamped to it
    _, big = mask_call(masks, bi[:2], stride, (H * stride + 37, W * stride + 5), out_hw)
    _, clamped = mask_call(masks, bi[:2], stride, (H * stride, W * stride), out_hw)
    assert torch.equal(big.view, clamped.view)


@gpu
@pytest.mark.parametrize("ow,shift", [(64, 0), (65, 0), (66, 0), (67, 0), (64, 1), (67, 3)])
def test_mask_chain_both_store_paths(ow, shift):
    g = torch.Generator(device="cuda").manual_seed(ow + shift)
    masks = torch.randn(5, 16, 16, device="cuda", generator=g) * 4
    bi = torch.tensor([3, 0, 4], device="cuda")
    got = mask_check(masks, bi, 4, (60, 64), (37, ow), f"ow={ow} shift={shift}", shift=shift)
    if shift == 0 and ow == 64:
        _, off = mask_call(masks, bi, 4, (60, 64), (37, ow), shift=1)
        assert torch.equal(off.view, got), "the scalar store path differs from the uchar4 path"


@gpu
def test_mask_chain_exact_probes():
    H, W, stride, crop, out_hw = 24, 20, 4, (90, 77), (131, 97)
    g = torch.Generator(device="cuda").manual_seed(2)
    mag = 0.25 + torch.rand(3, H, W, device="cuda", generator=g) * 4
    bi = torch.tensor([0, 1, 2], device="cuda")
    _, pos = mask_call(mag, bi, stride, crop, out_hw)
    _, neg = mask_call(-mag, bi, stride, crop, out_hw)
    assert bool((pos.view == 1).all()) and bool((neg.view == 0).all())
    # linear ramps across the columns and the rows, zero line between two source columns / rows: a pixel all of whose
    # source taps lie on one side is decided by that side, whatever the weights
    xs = torch.arange(W, device="cuda", dtype=torch.float32) - (W / 2 - 0.5)
    ys = torch.arange(H, device="cuda", dtype=torch.float32) - (H / 3 - 0.5)
    ramps = torch.stack([xs[None, :].expand(H, W), ys[:, None].expand(H, W), -xs[None, :].expand(H, W)]).contiguous()
    _, got = mask_call(ramps, bi, stride, crop, out_hw)
    cw, ch = min(crop[1], W * stride), min(crop[0], H * stride)

    def source_taps(n_src, n_mid, n_out, c):
        a0, a1, _, _ = mask_taps(mask_scale(c, n_out), n_out, c)             # output -> intermediate
        b0, b1, _, _ = mask_taps(mask_scale(n_src, n_mid), n_mid, n_src)     # intermediate -> source
        return torch.stack([b0[a0], b1[a0], b0[a1], b1[a1]], 1)              # [n_out, 4] source indices touched
    tx = source_taps(W, W * stride, out_hw[1], cw).cuda()
    ty = source_taps(H, H * stride, out_hw[0], ch).cuda()
    for r, (vals, taps, axis) in enumerate(((xs, tx, 1), (ys, ty, 0), (-xs, tx, 1))):
        tv = vals[taps]
        pos1, neg1 = (tv > 0).all(1), (tv < 0).all(1)
        plane = got.view[r]
        sel = plane if axis == 0 else plane.T                               # first index: the ramp's axis
        assert bool((sel[pos1] == 1).all()) and bool((sel[neg1] == 0).all()), f"ramp {r}"
        assert int(pos1.sum()) > 0 and int(neg1.sum()) > 0


@gpu
def test_mask_chain_rejections_leave_the_output_untouched():
    masks = torch.randn(2, 8, 8, device="cuda")
    bi = torch.zeros(65536, dtype=torch.int64, device="cuda")
    out = Canvas((65536, 1, 1), torch.uint8, pre=0xCD, fill=0xEE)      # a full-size output: a missed rejection is a value
    rc, _ = mask_call(masks, bi, 4, (32, 32), (1, 1), out=out)
    assert rc == EUNSUPPORTED
    out.untouched("num_det 65536")
    tall = Canvas((1, 262141, 1), torch.uint8, pre=0xCD, fill=0xEE)   # grid.y = 65536
    rc, _ = mask_call(masks, bi[:1], 4, (32, 32), (262141, 1), out=tall)
    assert rc == EUNSUPPORTED
    tall.untouched("out_h 262141")
    small = Canvas((1, 8, 8), torch.uint8, pre=0xCD, fill=0xEE)
    L = _lib.lib()
    for args in ((1, 0, 8, 4, 32, 32, 8, 8), (1, 8, 8, 0, 32, 32, 8, 8), (1, 8, 8, 4, 0, 32, 8, 8), (1, 8, 8, 4, 32, 32, 8, 0),
                 (-1, 8, 8, 4, 32, 32, 8, 8)):
        assert L.vllm_mask_postprocess_f32(masks.data_ptr(), bi.data_ptr(), *args, small.ptr, stream()) == EINVAL, args
    torch.cuda.synchronize()
    small.untouched("mask EINVAL")


# ---------------------------------------------------------------------------------------------------------------------
# 5. padded head stacking
# ---------------------------------------------------------------------------------------------------------------------
def hs_call(packed_ptr, ld, q, k, v, B, T, Tp, nq, nkv, D, to_stacked):
    rc = _lib.lib().vllm_head_stack_qkv_pad_bf16(packed_ptr, ld, q, k, v, B, T, Tp, nq, nkv, D, int(to_stacked), stream())
    torch.cuda.synchronize()
    return rc


@gpu
@pytest.mark.parametrize("B,T,Tp,nq,nkv,D", [(2, 300, 512, 4, 2, 64), (3, 1000, 1024, 8, 2, 128), (2, 77, 256, 2, 2, 64),
                                             (2, 300, 512, 4, 0, 64), (1, 256, 256, 3, 0, 8)])
def test_head_stack_qkv_pad_zero_rows_and_round_trip(B, T, Tp, nq, nkv, D):
    g = torch.Generator(device="cuda").manual_seed(T + nq)
    H = nq + 2 * nkv
    Wd = H * D
    ld = Wd + 16
    packed = Canvas((B, T, Wd), torch.bfloat16, ld=ld, pre=0.0)                 # NaN pitch gap: never read going out
    packed.buf.fill_(NAN)
    packed.view.copy_(torch.randn(B, T, Wd, device="cuda", generator=g).bfloat16())
    packed.before = bits(packed.buf).clone()
    stk = Canvas((H * B * Tp, D), torch.bfloat16)
    nq_rows, nkv_rows = B * nq * Tp, B * nkv * Tp
    q = stk.view[:nq_rows]
    k = stk.view[nq_rows:nq_rows + nkv_rows] if nkv else None
    v = stk.view[nq_rows + nkv_rows:] if nkv else None
    assert hs_call(packed.ptr, ld, q.data_ptr(), k.data_ptr() if nkv else None, v.data_ptr() if nkv else None,
                   B, T, Tp, nq, nkv, D, True) == OK
    packed.untouched("the packed rows going to the stacks")
    heads = packed.view.reshape(B, T, H, D).permute(2, 0, 1, 3)                # [H, B, T, D]
    want = torch.zeros((H, B, Tp, D), dtype=torch.bfloat16, device="cuda")
    want[:, :, :T] = heads
    # q stacks [B, nq, Tp, D], then k / v [B, nkv, Tp, D]
    order = [want[:nq].permute(1, 0, 2, 3).reshape(-1, D)]
    if nkv:
        order += [want[nq:nq + nkv].permute(1, 0, 2, 3).reshape(-1, D), want[nq + nkv:].permute(1, 0, 2, 3).reshape(-1, D)]
    stk.check(torch.cat(order), "stacks (pad rows +0)")
    # coming back: NaN in every pad row of the stacks, a NaN-prefilled packed output with a sentinel pitch gap
    back = Canvas((B, T, Wd), torch.bfloat16, ld=ld)
    st = stk.view.clone()
    st.view(-1, Tp, D)[:, T:] = NAN
    qb = st[:nq_rows]
    kb = st[nq_rows:nq_rows + nkv_rows] if nkv else None
    vb = st[nq_rows + nkv_rows:] if nkv else None
    assert hs_call(back.ptr, ld, qb.data_ptr(), kb.data_ptr() if nkv else None, vb.data_ptr() if nkv else None,
                   B, T, Tp, nq, nkv, D, False) == OK
    back.check(packed.view, "round trip (NaN pad rows not read)")
    # rejections: tokens_pad < tokens, nq % nkv, head_dim % 8, ld % 8
    bad = Canvas((H * B * Tp, D), torch.bfloat16)
    for args, want_rc in (((B, T, T - 1, nq, nkv, D), EINVAL), ((B, T, Tp, nq + 1, max(nkv, 2), D), EINVAL),
                          ((B, T, Tp, nq, nkv, D - 4), EUNSUPPORTED), ((B, T, Tp, nq, nkv, 4), EUNSUPPORTED)):
        assert hs_call(packed.ptr, ld, bad.ptr, bad.ptr, bad.ptr, *args, True) == want_rc, args
    assert hs_call(packed.ptr, ld + 4, bad.ptr, bad.ptr, bad.ptr, B, T, Tp, nq, nkv, D, True) == EALIGN
    if nkv:                                                          # the unpadded form rejects head_dim < 8 the same way
        assert _lib.lib().vllm_head_stack_qkv_bf16(packed.ptr, ld, bad.ptr, bad.ptr, bad.ptr, B, T, nq, nkv, 4, 1,
                                                   stream()) == EUNSUPPORTED
    torch.cuda.synchronize()
    bad.untouched("head_stack rejections")
    packed.untouched("head_stack rejections")
