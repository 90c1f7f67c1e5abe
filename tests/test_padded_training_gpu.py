"""GPU: the multimodal chat training step on right-padded batches (visionllm_b200/train.py, csrc/train_ops.cu) -- the
length-masked causal softmax, the padded attention backward, the bridge and sequence-assembly backward kernels, the
decoder with an attention mask and the composite `B200VisionLLMv2ModelTrain` step.

Checkers are those of tests/test_train_kernels_contract_gpu.py (`rounds` / `within` of tests/bf16_rounding.py, no
max|ref| term).  Bounds stated here, u = 2^-24:
  length softmax  the causal softmax bound over the visible keys j <= i, j < len (the same kernel and reduction order).
  GELU            y = gelu(u) within 16u (|z| + |u| / 2); dx = dy gelu'(u) within |dy| (16u (Phi(u) + |u| phi(u) (1 + u^2))
                  + 4u) (erff / expf within 2 ulp of their fp32 arguments, a few fp32 roundings; the absolute 4u is
                  1 + erf(u / sqrt 2) cancelling for negative u, where Phi(u) and u phi(u) nearly cancel too).
  bias grad       fp32 sums of bf16 dy: c u sum|dy|, c = rows_per_cta + ceil(n_partials / 8) + 10 (the per-CTA chain, the
                  8-warp partial chain and tree).
  LN dweight      sum dy xhat with xhat = (x - mean) rstd from fp32 statistics: c u sum|dy xhat| plus sum|dy| (|xhat| er +
                  rstd d u mean|x|), d = 8 VPT + 13, er = (d / 2 + 6) u; dbias as the bias gradient.
  modules         rel_l2(ours, fp32 ref) <= 2 rel_l2(bf16 ref, fp32 ref) + 3e-3 (the existing module rule).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bf16_rounding import U, note_ratio, print_report, rn_bf16, rounds, within
from test_train_kernels_contract_gpu import (EALIGN, EINVAL, NAN, bits, causal_stack, f32, gen, regions, same_bits,
                                             softmax_call, vpt)
from visionllm_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("padded training step")


def stream():
    return torch.cuda.current_stream().cuda_stream


def rel(a, b):
    return float(torch.linalg.norm((a.double() - b.double()).flatten()) / (torch.linalg.norm(b.double().flatten()) + 1e-300))


def len_call(s, n_mat, hpb, T, lens, scale):
    return _lib.lib().vllm_softmax_causal_len_bf16(s.data_ptr(), s.stride(0), n_mat, hpb, T, lens.data_ptr(), scale, stream())


# ---------------------------------------------------------------------------------------------------------------------
# length softmax
# ---------------------------------------------------------------------------------------------------------------------
def visible(T, lens, hpb):
    """[n_mat, T, T]: key j visible to query i of matrix m iff j <= i and j < lens[m // hpb]."""
    i = torch.arange(T, device="cuda")[:, None]
    j = torch.arange(T, device="cuda")[None, :]
    L = lens.long().repeat_interleave(hpb)[:, None, None]
    return (j <= i)[None] & (j < L)


@pytest.mark.parametrize("T", [256, 1024, 2304])
def test_length_softmax_vs_fp64(T):
    """P against fp64 over the visible keys; NaN in S above the diagonal and at every masked key: exact 0 there inside the
    diagonal block, nothing beyond it written."""
    g = gen(T + 7)
    hpb, nb = 2, 3
    n_mat, ld = hpb * nb, T + 16
    lens = torch.tensor([1, T, T * 3 // 5 + 3], dtype=torch.int32, device="cuda")
    low, zero, keep = regions(T, ld)
    vis = visible(T, lens, hpb)
    d = 8 * vpt(T) + 13
    sf = f32(128 ** -0.5)
    vals = (torch.randn(n_mat, T, T, device="cuda", generator=g) * 4).bfloat16()
    s = causal_stack(torch.where(vis, vals, torch.full_like(vals, NAN)), T, ld, low)
    before = s.clone()
    assert len_call(s, n_mat, hpb, T, lens, 128 ** -0.5) == 0
    torch.cuda.synchronize()
    o = s.view(n_mat, T, ld)
    p = o[:, :, :T]
    written = (low | zero)[:, :T][None].expand(n_mat, -1, -1)
    assert (p[written & ~vis] == 0).all(), "masked keys inside the written block are not exact 0"
    assert torch.equal(bits(o)[:, keep], bits(before.view(n_mat, T, ld))[:, keep]), "wrote beyond the diagonal block"
    v = torch.where(vis, vals.double() * sf, torch.full((), -math.inf, dtype=torch.float64, device="cuda"))
    mx = v.amax(-1, keepdim=True)
    x = v - mx
    z = torch.softmax(v, -1)
    e = torch.where(vis, 2.0 ** -21 + x.abs() * 2.0 ** -23 + U * (v.abs() + mx.abs() + x.abs()), torch.zeros_like(v))
    E = 1.25 * z * (e + e.amax(-1, keepdim=True) + (d + 3) * U)
    rounds(p[vis], z[vis], E[vis], "softmax_causal_len", f"T={T}")


@pytest.mark.parametrize("T", [256, 2304])
def test_length_softmax_probes_and_identity(T):
    """Key-count probe: P = RN_bf16(fl32(1 / min(i + 1, len))) on the visible keys.  lens == T is bit-identical to
    vllm_softmax_causal_bf16, NaN-free and NaN-filled above the diagonal alike."""
    hpb, n_mat, ld = 1, 3, T + 8
    lens = torch.tensor([5, T, 130], dtype=torch.int32, device="cuda")
    low, zero, keep = regions(T, ld)
    vis = visible(T, lens, hpb)
    s = causal_stack(torch.where(vis, torch.full((n_mat, T, T), 0.75, dtype=torch.bfloat16, device="cuda"),
                                 torch.full((), NAN, dtype=torch.bfloat16, device="cuda")), T, ld, low)
    assert len_call(s, n_mat, hpb, T, lens, 0.1) == 0
    torch.cuda.synchronize()
    cnt = torch.minimum(torch.arange(1, T + 1, device="cuda")[None, :], lens.long()[:, None])        # [n_mat, T]
    inv = torch.from_numpy(np.float32(1) / np.arange(1, T + 1, dtype=np.float32)).cuda().double()
    want = rn_bf16(inv[cnt - 1])[:, :, None].expand(n_mat, T, T)
    p = s.view(n_mat, T, ld)[:, :, :T].double()
    assert torch.equal(p[vis], want[vis]), "key-count probe: P != bf16(1 / min(i + 1, len))"
    g = gen(T)
    vals = (torch.randn(4, T, T, device="cuda", generator=g) * 3).bfloat16()
    a = causal_stack(vals, T, ld, low)
    b = a.clone()
    full = torch.full((2,), T, dtype=torch.int32, device="cuda")
    assert softmax_call(a, 4, T, 0.125) == 0 and len_call(b, 4, 2, T, full, 0.125) == 0
    torch.cuda.synchronize()
    assert same_bits(a, b), "lens == T differs from vllm_softmax_causal_bf16"


def test_length_softmax_rejections_leave_the_buffer_untouched():
    L = _lib.lib()
    st = stream()
    s = torch.full((512, 264), 1.0, dtype=torch.bfloat16, device="cuda")
    lens = torch.full((2,), 256, dtype=torch.int32, device="cuda")
    before = s.clone()
    sp, lp = s.data_ptr(), lens.data_ptr()
    assert L.vllm_softmax_causal_len_bf16(sp, 264, 2, 0, 256, lp, 0.1, st) == EINVAL       # heads_per_batch
    assert L.vllm_softmax_causal_len_bf16(sp, 264, 2, 3, 256, lp, 0.1, st) == EINVAL       # n_mat % heads_per_batch
    assert L.vllm_softmax_causal_len_bf16(sp, 264, 2, 1, 256, None, 0.1, st) == EINVAL     # no lengths
    assert L.vllm_softmax_causal_len_bf16(sp, 264, 2, 1, 252, lp, 0.1, st) == EINVAL       # T % 8
    assert L.vllm_softmax_causal_len_bf16(sp, 248, 2, 1, 256, lp, 0.1, st) == EINVAL       # ld < T
    assert L.vllm_softmax_causal_len_bf16(sp + 2, 264, 2, 1, 256, lp, 0.1, st) == EALIGN
    torch.cuda.synchronize()
    assert same_bits(s, before)


# ---------------------------------------------------------------------------------------------------------------------
# padded attention backward
# ---------------------------------------------------------------------------------------------------------------------
def masked_attention_grads(qkv5, do, scale, lens, dtype):
    """d(qkv5) of HF eager attention with the causal + key-length mask (repeat_kv, scores in `dtype`, fp32 softmax)."""
    B, T, P, nkv, D = qkv5.shape
    G = P - 2
    t = qkv5.detach().to(dtype).requires_grad_(True)
    q = t[:, :, :G].reshape(B, T, G * nkv, D).transpose(1, 2)
    k = t[:, :, G].transpose(1, 2).repeat_interleave(G, 1)
    v = t[:, :, G + 1].transpose(1, 2).repeat_interleave(G, 1)
    s = torch.matmul(q, k.transpose(2, 3)) * scale
    i = torch.arange(T, device="cuda")
    blocked = (i[None, :] > i[:, None])[None] | (i[None, None, :] >= lens.long()[:, None, None])       # [B, T, T]
    s = s.masked_fill(blocked[:, None], torch.finfo(dtype).min)
    p = torch.softmax(s, -1, dtype=torch.float32 if dtype != torch.float64 else dtype).to(dtype)
    o = torch.matmul(p, v).transpose(1, 2).reshape(B, T, G * nkv * D)
    o.backward(do.to(dtype))
    return t.grad


@pytest.mark.parametrize("G", [1, 6])
def test_padded_backward_all_valid_is_bit_identical(G):
    """T % 256 == 0 and every key valid: the length path equals today's attention_backward_packed bit for bit."""
    from visionllm_b200 import train as TR
    B, T, D = 2, 512, 128
    nkv = 2 if G == 1 else 1
    g = gen(G)
    qkv5 = (torch.randn(B, T, G + 2, nkv, D, device="cuda", generator=g) * 0.5).bfloat16()
    do = (torch.randn(B, T, G * nkv * D, device="cuda", generator=g) * 0.5).bfloat16()
    a = TR.attention_backward_packed(qkv5, do, D ** -0.5)
    b = TR.attention_backward_packed(qkv5, do, D ** -0.5, torch.full((B,), T, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert same_bits(a, b)


@pytest.mark.parametrize("G", [1, 6])
@pytest.mark.parametrize("T", [1, 200, 300, 777, 1024])
def test_padded_backward_vs_fp64(T, G):
    """Ragged lengths (1, full, mixed) against fp64 autograd of the masked attention, module rule."""
    from visionllm_b200 import train as TR
    D = 64
    nkv = 2 if G == 1 else 1
    lens = torch.tensor(sorted({1, T, max(1, T // 3 + 1)}), dtype=torch.int32, device="cuda")
    B = lens.numel()
    g = gen(T * 10 + G)
    qkv5 = (torch.randn(B, T, G + 2, nkv, D, device="cuda", generator=g) * 0.5).bfloat16()
    do = (torch.randn(B, T, G * nkv * D, device="cuda", generator=g) * 0.5).bfloat16()
    got = TR.attention_backward_packed(qkv5, do, D ** -0.5, lens)
    assert not got.isnan().any()
    ref = masked_attention_grads(qkv5, do, D ** -0.5, lens, torch.float64)
    bf = masked_attention_grads(qkv5, do, D ** -0.5, lens, torch.bfloat16)
    for name, sl in (("dq", slice(0, G)), ("dk", slice(G, G + 1)), ("dv", slice(G + 1, G + 2))):
        a, b = rel(got[:, :, sl], ref[:, :, sl]), rel(bf[:, :, sl], ref[:, :, sl])
        note_ratio("padded_attention_bwd_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (name, T, G, a, b)
    for b_, n in enumerate(lens.tolist()):                       # keys past the length take no gradient
        assert (got[b_, n:, G:] == 0).all()


@pytest.mark.parametrize("G", [1, 6])
def test_padded_row_equals_the_sequence_alone_and_ignores_padding(G):
    """Row 0 of a padded batch with zero dO past its length equals that sequence run alone (up to the sign of zero):
    past the length dO = 0 gives dP = 0, so dS = 0 there, and the extra k-blocks of the GEMMs add exact zeros in the same
    order.  Finite garbage in the padded K / V rows changes nothing."""
    from visionllm_b200 import train as TR
    D, T, n0 = 64, 700, 333
    nkv = 2 if G == 1 else 1
    g = gen(G + 99)
    qkv5 = (torch.randn(2, T, G + 2, nkv, D, device="cuda", generator=g) * 0.5).bfloat16()
    do = (torch.randn(2, T, G * nkv * D, device="cuda", generator=g) * 0.5).bfloat16()
    do[0, n0:] = 0
    lens = torch.tensor([n0, T], dtype=torch.int32, device="cuda")
    got = TR.attention_backward_packed(qkv5, do, D ** -0.5, lens)
    alone = TR.attention_backward_packed(qkv5[:1, :n0].contiguous(), do[:1, :n0].contiguous(), D ** -0.5)
    torch.cuda.synchronize()
    assert torch.equal(got[0, :n0].float(), alone[0].float()), "row 0 differs from the sequence run alone"
    assert (got[0, n0:] == 0).all()
    dirty = qkv5.clone()
    dirty[0, n0:, G:] = (torch.randn(T - n0, 2, nkv, D, device="cuda", generator=g) * 50).bfloat16()
    got2 = TR.attention_backward_packed(dirty, do, D ** -0.5, lens)
    torch.cuda.synchronize()
    assert same_bits(got2[0, :n0], got[0, :n0]) and same_bits(got2[1], got[1]), "padded K / V rows leaked"


# ---------------------------------------------------------------------------------------------------------------------
# bridge kernels
# ---------------------------------------------------------------------------------------------------------------------
def chain_c(rows):
    n_part = _lib.lib().vllm_rmsnorm_bwd_partials(rows)
    rpc = -(-rows // n_part)
    return rpc + -(-n_part // 8) + 10


@pytest.mark.parametrize("cols", [256, 4096, 12800])
def test_gelu_forward_backward_vs_fp64(cols):
    from visionllm_b200 import train as TR
    g = gen(cols)
    rows = 67
    u = (torch.randn(rows, cols, device="cuda", generator=g) * 3).bfloat16()
    u[0, :8] = torch.tensor([0, -0.0, 1e-30, -1e-30, 10, -10, 40, -40], dtype=torch.bfloat16)
    dy = (torch.randn(rows, cols, device="cuda", generator=g)).bfloat16()
    ud, dd = u.double(), dy.double()
    Phi = 0.5 * (1 + torch.erf(ud / math.sqrt(2)))
    phi = torch.exp(-0.5 * ud * ud) / math.sqrt(2 * math.pi)
    y = TR.gelu_fwd(u)
    z = ud * Phi
    rounds(y, z, 16 * U * (z.abs() + 0.5 * ud.abs()), "gelu_fwd", f"cols={cols}")
    dx = TR.gelu_bwd(u, dy)
    z = dd * (Phi + ud * phi)
    rounds(dx, z, dd.abs() * (16 * U * (Phi + ud.abs() * phi * (1 + ud * ud)) + 4 * U), "gelu_bwd", f"cols={cols}")
    assert same_bits(TR.gelu_bwd(u, dy), dx) and same_bits(TR.gelu_fwd(u), y)
    assert (TR.gelu_bwd(u, torch.zeros_like(dy)) == 0).all()


@pytest.mark.parametrize("rows,cols", [(1, 8), (300, 4096), (4100, 768), (2048, 12800)])
def test_bias_and_layernorm_grads_vs_fp64(rows, cols):
    from visionllm_b200 import train as TR
    g = gen(rows + cols)
    dy = (torch.randn(rows, cols, device="cuda", generator=g)).bfloat16()
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 2 + 0.5).bfloat16()
    c = chain_c(rows)
    db = TR.bias_grad(dy)
    dd = dy.double()
    within(db, dd.sum(0), c * U * dd.abs().sum(0), "bias_grad", f"{rows}x{cols}")
    eps = 1e-6
    dw, db2 = TR.layernorm_bwd_wb(x, dy, eps)
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(((xd - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = (xd - mean) * rstd
    d = 8 * (1 if cols // 8 <= 256 else 2 if cols // 8 <= 512 else 4 if cols // 8 <= 1024 else 8) + 13
    er = (d / 2 + 6) * U
    E = c * U * (dd * xh).abs().sum(0) + (dd.abs() * (xh.abs() * er + rstd * d * U * xd.abs().mean(-1, keepdim=True))).sum(0)
    within(dw, (dd * xh).sum(0), E, "layernorm_dweight", f"{rows}x{cols}")
    within(db2, dd.sum(0), c * U * dd.abs().sum(0), "layernorm_dbias", f"{rows}x{cols}")
    # run-to-run identical; exact probes
    assert same_bits(TR.bias_grad(dy), db) and same_bits(TR.layernorm_bwd_wb(x, dy, eps)[0], dw)
    zero = torch.zeros_like(dy)
    assert (TR.bias_grad(zero) == 0).all() and all((t == 0).all() for t in TR.layernorm_bwd_wb(x, zero, eps))
    ones = torch.ones_like(dy)
    assert (TR.bias_grad(ones) == rows).all()                   # integer sums below 2^24 are exact
    const = torch.full_like(x, 1.5)                             # constant rows: xhat = 0
    dwc, dbc = TR.layernorm_bwd_wb(const, ones, eps)
    assert (dwc == 0).all() and (dbc == rows).all()


# ---------------------------------------------------------------------------------------------------------------------
# sequence assembly backward
# ---------------------------------------------------------------------------------------------------------------------
def test_assemble_embeds_backward_vs_index_add():
    from visionllm_b200 import ops, train as TR
    V, C, E_, IMP, EMB, DET, POSE = 500, 256, 4, 400, 490, 410, 420
    B, L = 3, 300
    g = gen(5)
    ids = torch.randint(0, 380, (B, L), device="cuda", generator=g)
    ids[0, 10:42] = IMP                                          # 32 image tokens per sample, samples 0 and 2
    ids[2, 100:132] = IMP
    for b, p, t in ((0, 60, DET), (1, 7, DET), (1, 200, POSE), (2, 250, DET)):
        ids[b, p] = t
        ids[b, p + 1:p + 1 + E_] = EMB + torch.arange(E_, device="cuda")
    plan = ops.seq_index(ids, (DET,), (POSE,), EMB, E_, IMP, None, 32)
    assert int(plan.status.item()) == 0
    n_img = B * 32                                               # sample 1 has no image tokens: its rows are unplaced
    dy = torch.randn(B, L, C, device="cuda", generator=g).bfloat16()
    outs = TR.assemble_embeds_bwd(plan, dy, (V, E_, E_, n_img), [True] * 4)
    again = TR.assemble_embeds_bwd(plan, dy, (V, E_, E_, n_img), [True] * 4)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(outs, again)), "not run-to-run identical"
    kind, row = plan.kind.reshape(-1).long(), plan.row.reshape(-1).long()
    flat = dy.reshape(-1, C).double()
    for k, (n, got) in enumerate(zip((V, E_, E_, n_img), outs)):
        sel = kind == k
        ref = torch.zeros((n, C), dtype=torch.float64, device="cuda").index_add_(0, row[sel], flat[sel])
        absr = torch.zeros((n, C), dtype=torch.float64, device="cuda").index_add_(0, row[sel], flat[sel].abs())
        cnt = torch.bincount(row[sel], minlength=n).double()[:, None]
        if k == 3:
            assert torch.equal(got.double(), ref), "image-feature gather is not exact"
        else:
            rounds(got, ref, cnt * U * absr, "assemble_bwd_tables", f"source {k}")
        assert (got[cnt[:, 0] == 0] == 0).all(), f"source {k}: unreferenced rows not exact 0"
    assert (outs[3][32:64] == 0).all()                          # the image rows of sample 1 were never placed
    part = TR.assemble_embeds_bwd(plan, dy, (V, E_, E_, n_img), [False, True, False, True])
    assert part[0] is None and part[2] is None and same_bits(part[1], outs[1]) and same_bits(part[3], outs[3])


# ---------------------------------------------------------------------------------------------------------------------
# decoder with padding
# ---------------------------------------------------------------------------------------------------------------------
def padded_batch(B, T, H, V, lens, seed):
    gen_ = torch.Generator().manual_seed(seed)
    emb = (torch.randn(B, T, H, generator=gen_) * 0.5).bfloat16()
    labels = torch.randint(0, V, (B, T), generator=gen_)
    mask = (torch.arange(T)[None] < torch.tensor(lens)[:, None]).long()
    labels[mask == 0] = -100
    labels[:, :20] = -100
    return emb, labels, mask


@pytest.mark.parametrize("nkv", [4, 2], ids=["mha", "gqa"])
@pytest.mark.parametrize("T", [200, 512])
def test_llama_decoder_with_padding_matches_hf(T, nkv):
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    H, V = 256, 1000
    cfg = LlamaConfig(hidden_size=H, intermediate_size=688, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=nkv, vocab_size=V, rms_norm_eps=1e-5, max_position_embeddings=1024,
                      attn_implementation="eager")
    torch.manual_seed(nkv)
    hf = LlamaForCausalLM(cfg)
    sd = {k: v.to(torch.bfloat16).float() for k, v in hf.state_dict().items()}
    hf.load_state_dict(sd)
    lens = [T, T // 2 + 1, 37]
    B = len(lens)
    emb, labels, mask = padded_batch(B, T, H, V, lens, T + nkv)

    def hf_run(dtype):
        m = hf.to("cuda", dtype).train(False)
        for p in m.parameters():
            p.grad = None
        e = emb.to("cuda", dtype).requires_grad_(True)
        logits = m(inputs_embeds=e, attention_mask=mask.cuda()).logits.float()
        loss = F.cross_entropy(logits[:, :-1].reshape(-1, V), labels.cuda()[:, 1:].reshape(-1), ignore_index=-100)
        loss.backward()
        return float(loss.detach()), e.grad.float(), {n: p.grad.float().clone() for n, p in m.named_parameters() if p.grad is not None}

    l64, de64, g64 = hf_run(torch.float64)
    l16, de16, g16 = hf_run(torch.bfloat16)
    mine = B200LlamaForCausalLM(cfg)
    mine.load_state_dict(sd)
    mine = mine.to("cuda", torch.bfloat16)
    tr = B200LlamaForCausalLMTrain(mine)
    e = emb.cuda().requires_grad_(True)
    loss, _, _ = tr(e, labels.cuda(), attention_mask=mask.cuda())
    loss.backward()
    assert abs(float(loss) - l64) <= 1.5 * abs(l16 - l64) + 1e-3 * abs(l64), (float(loss), l64, l16)
    a, b = rel(e.grad, de64), rel(de16, de64)
    note_ratio("decoder_padded_module_rule", a / (2 * b + 3e-3))
    assert a <= 2 * b + 3e-3, ("inputs_embeds", a, b)
    for n, p in mine.named_parameters():
        if n == "model.embed_tokens.weight":
            continue
        a, b = rel(p.grad, g64[n]), rel(g16[n], g64[n])
        note_ratio("decoder_padded_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (n, a, b)


def test_internlm2_decoder_with_padding_matches_reference_golden():
    """B200InternLM2ForCausalLMTrain (48-over-8-style grouped-query heads: 12 over 2 here) with a right-padded, ragged
    attention_mask at T = 200 against tests/golden/train_internlm2_padded.npz -- the reference's own InternLM2ForCausalLM
    with its own 4-D mask, fp32 and bf16 autograd on CPU: module rule on the loss, the logits of valid positions, the input
    gradient and every parameter gradient."""
    import json
    import os
    import sys
    from types import SimpleNamespace
    from test_gqa_backward_gpu import ROOT, module_rule
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from train_internlm2_padded_inputs import WEIGHT_SEED, checksum, inputs
    from weights_util import key_shapes, seeded_state_dict
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    gz = np.load(os.path.join(ROOT, "tests", "golden", "train_internlm2_padded.npz"))
    cfg = SimpleNamespace(rope_scaling=None, hidden_act="silu", bias=False, pad_token_id=None, **json.loads(str(gz["config"])))
    lm = B200InternLM2ForCausalLM(cfg)
    assert json.loads(str(gz["keys"])) == [list(k) for k in key_shapes(lm)]
    lm.load_state_dict(seeded_state_dict(lm, WEIGHT_SEED))
    lm = lm.to("cuda", torch.bfloat16)
    tr = B200InternLM2ForCausalLMTrain(lm)
    emb, labels, mask = inputs()
    assert torch.equal(checksum(emb, labels), torch.from_numpy(gz["inputs_checksum"])) and (mask.numpy() == gz["mask"]).all()
    e = emb.cuda().bfloat16().requires_grad_(True)
    loss, logits, _ = tr(e, labels.cuda(), attention_mask=mask.cuda())
    loss.backward()
    assert (e.grad[mask.cuda() == 0] == 0).all()

    def sample(key, t):
        idx = torch.from_numpy(gz[key + "/idx"]).long().cuda()
        return (t.detach().float().reshape(-1)[idx], torch.from_numpy(gz[key + "/f32"]).cuda(),
                torch.from_numpy(gz[key + "/refbf16"]).cuda())

    named = dict(lm.named_parameters())
    names = json.loads(str(gz["params"]))
    assert all(named[n].grad is not None for n in names)
    params = {n: sample("grad/" + n, named[n].grad) for n in names}
    for n, (a_, r32, r16) in params.items():
        note_ratio("decoder_padded_module_rule", rel(a_, r32) / (2 * rel(r16, r32) + 3e-3))
    module_rule((float(loss.detach()), float(gz["loss_f32"]), float(gz["loss_refbf16"])),
                sample("logits", logits), sample("d_emb", e.grad), params)


def test_all_ones_mask_takes_the_unmasked_path():
    from transformers import LlamaConfig
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    cfg = LlamaConfig(hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=1000, rms_norm_eps=1e-5)
    torch.manual_seed(1)
    mine = B200LlamaForCausalLM(cfg).to("cuda", torch.bfloat16)
    tr = B200LlamaForCausalLMTrain(mine)
    emb, labels, mask = padded_batch(2, 256, 256, 1000, [256, 256], 4)
    grads = []
    for m in (None, mask.cuda()):
        for p in mine.parameters():
            p.grad = None
        e = emb.cuda().requires_grad_(True)
        loss, _, _ = tr(e, labels.cuda(), attention_mask=m)
        loss.backward()
        grads.append([e.grad] + [p.grad for p in mine.parameters() if p.grad is not None])
    assert all(same_bits(a, b) for a, b in zip(*grads))


# ---------------------------------------------------------------------------------------------------------------------
# the composite step
# ---------------------------------------------------------------------------------------------------------------------
V_, IMP_, EMB_, DET_, POSE_, NE_ = 1000, 980, 990, 970, 975, 4


def build_composite(bridge, pixelshuffle):
    from types import SimpleNamespace
    from transformers import LlamaConfig
    from visionllm_b200.internvit import B200InternVisionModel, InternVisionConfig
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.modeling import B200VisionLLMv2Model
    torch.manual_seed(11)
    vit = B200InternVisionModel(InternVisionConfig(hidden_size=192, num_attention_heads=3, num_hidden_layers=2,
                                                   intermediate_size=768, image_size=112, patch_size=14))
    llm = B200LlamaForCausalLM(LlamaConfig(hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                                           num_attention_heads=4, num_key_value_heads=4, vocab_size=V_, rms_norm_eps=1e-5,
                                           pad_token_id=0))
    cfg = SimpleNamespace(use_pixelshuffle=pixelshuffle, vl_bridge_type=bridge, vis_output_layer=-1, num_embs=NE_,
                          imp_token_id=IMP_, emb_token_id=EMB_, det_tool_id=DET_, seg_tool_id=-1, grd_tool_id=-1,
                          pose_tool_id=POSE_)
    m = B200VisionLLMv2Model(cfg, vit, llm)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.copy_(torch.randn_like(p) * (0.05 if p.dim() > 1 else 0.2) + (1.0 if n.endswith("norm.weight") or
                                                                            n.endswith("layernorm.weight") else 0.0))
    return m.to("cuda", torch.bfloat16)


def composite_batch(n_img_tokens, L=230):
    g = torch.Generator().manual_seed(21)
    lens = [L, 171]
    ids = torch.randint(1, 900, (2, L), generator=g)
    for b in range(2):
        ids[b, 5:5 + n_img_tokens] = IMP_
        p = 5 + n_img_tokens + 10
        ids[b, p] = DET_ if b == 0 else POSE_
        ids[b, p + 1:p + 1 + NE_] = EMB_ + torch.arange(NE_)
    ids[1, lens[1]:] = 0                                        # the pad id, also at some valid positions (unk)
    ids[:, 150:153] = 0
    mask = (torch.arange(L)[None] < torch.tensor(lens)[:, None]).long()
    labels = ids.clone()
    labels[:, :5 + n_img_tokens] = -100
    labels[mask == 0] = -100
    images = torch.randn(2, 3, 112, 112, generator=g)
    return ids, mask, labels, images


def reference_step(m, ids, mask, labels, images, dtype):
    """The chat step as a plain torch autograd composition in VisionLLMv2Model.forward's order (mv2.py:559-605, 724-757):
    frozen ViT features -> bridge -> embedding lookup, [EMB] table rows after the tool tokens, image features at the
    <im_patch> slots -> HF Llama with the attention mask -> shifted CE with the [EMB] labels ignored."""
    import torch.nn as nn
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200.modeling import BridgeLayerNorm, BridgeLinear, pixel_shuffle
    with torch.no_grad():
        hs, _, _ = m.vision_hidden_state(images.cuda().bfloat16())
    feats = hs[:, 1:].to(dtype)
    if m.use_pixelshuffle:
        h = int(feats.shape[1] ** 0.5)
        feats = pixel_shuffle(feats.reshape(feats.shape[0], h, h, -1), 0.5).reshape(feats.shape[0], -1, feats.shape[-1] * 4)
    params = {}

    def P(name, t):                                              # a leaf copy of parameter `name` in `dtype`
        params[name] = t.detach().to(dtype).requires_grad_(True)
        return params[name]

    mods = [m.vl_bridge] if isinstance(m.vl_bridge, BridgeLinear) else list(m.vl_bridge)
    x = feats
    for i, mod in enumerate(mods):
        pre = "vl_bridge." if len(mods) == 1 else f"vl_bridge.{i}."
        if isinstance(mod, BridgeLinear):
            x = F.linear(x, P(pre + "weight", mod.weight), P(pre + "bias", mod.bias))
        elif isinstance(mod, BridgeLayerNorm):
            x = F.layer_norm(x, (x.shape[-1],), P(pre + "weight", mod.weight), P(pre + "bias", mod.bias), mod.eps)
        elif isinstance(mod, nn.GELU):
            x = F.gelu(x)
    ids = ids.cuda()
    table = P("llm.model.embed_tokens.weight", m.llm.model.embed_tokens.weight)
    det, pose = P("emb_embeddings_det.weight", m.emb_embeddings_det.weight), P("emb_embeddings_pose.weight", m.emb_embeddings_pose.weight)
    emb = F.embedding(ids, table, padding_idx=0)               # the reference's nn.Embedding(..., padding_idx=pad_token_id)
    for tool, tab in ((DET_, det), (POSE_, pose)):
        b, p = torch.nonzero(ids == tool, as_tuple=True)
        for j in range(NE_):
            emb = emb.index_put((b, p + 1 + j), tab[j].expand(b.numel(), -1))
    emb = emb.index_put(torch.nonzero(ids == IMP_, as_tuple=True), x.reshape(-1, x.shape[-1]))
    lcfg = m.llm.config
    hf = LlamaForCausalLM(LlamaConfig(**{**lcfg.to_dict(), "attn_implementation": "eager"})).to("cuda", dtype)
    hf.load_state_dict({k: v.to(dtype) for k, v in m.llm.state_dict().items()}, strict=False)
    hf_params = dict(hf.named_parameters())
    for n, p in hf_params.items():
        if n != "model.embed_tokens.weight":
            params["llm." + n] = p
    logits = hf(inputs_embeds=emb, attention_mask=mask.cuda()).logits.float()
    lab = labels.clone().cuda()
    lab[(lab >= EMB_) & (lab < EMB_ + NE_)] = -100
    loss = F.cross_entropy(logits[:, :-1].reshape(-1, V_), lab[:, 1:].reshape(-1), ignore_index=-100)
    loss.backward()
    return float(loss), {k: v.grad for k, v in params.items()}


@pytest.mark.parametrize("bridge,pixelshuffle", [("linear", False), ("mlp2x_gelu", False), ("internvl_mlp", True)])
def test_composite_step_matches_torch_composition(bridge, pixelshuffle):
    from visionllm_b200.train import B200VisionLLMv2ModelTrain
    m = build_composite(bridge, pixelshuffle)
    m.freeze_vis_encoder()
    n_tok = 16 if pixelshuffle else 64
    ids, mask, labels, images = composite_batch(n_tok)
    l64, g64 = reference_step(m, ids, mask, labels, images, torch.float64)
    l16, g16 = reference_step(m, ids, mask, labels, images, torch.bfloat16)
    tr = B200VisionLLMv2ModelTrain(m)
    out = tr(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=images.cuda().bfloat16(), labels=labels.clone().cuda())
    out.loss.backward()
    assert abs(float(out.loss) - l64) <= 1.5 * abs(l16 - l64) + 1e-3 * abs(l64), (float(out.loss), l64, l16)
    named = dict(m.named_parameters())
    assert set(g64) <= set(named)
    for n, ref in g64.items():
        got = named[n].grad
        assert got is not None, n
        a, b = rel(got, ref), rel(g16[n], ref)
        note_ratio("composite_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (bridge, n, a, b)
    assert all(p.grad is None for p in m.vis_encoder.parameters())
    assert (named["llm.model.embed_tokens.weight"].grad[0] == 0).all()


def test_composite_freezing_and_refusals():
    from visionllm_b200.train import B200VisionLLMv2ModelTrain
    m = build_composite("mlp2x_gelu", False)
    m.freeze_vis_encoder()
    m.freeze_llm()
    m.freeze_emb_embeddings()
    ids, mask, labels, images = composite_batch(64)
    tr = B200VisionLLMv2ModelTrain(m)
    kw = dict(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=images.cuda().bfloat16(), labels=labels.clone().cuda())
    tr(**kw).loss.backward()
    for n, p in m.named_parameters():
        assert (p.grad is not None) == n.startswith("vl_bridge."), n
    for bad in (dict(targets=[{}]), dict(images_aug=[images[0]]), dict(regions=[torch.ones(1, 112, 112)]),
                dict(past_key_values=((),)), dict(images=images.cuda().float()), dict(inputs_embeds=torch.zeros(1))):
        with pytest.raises(NotImplementedError):
            tr(**{**kw, **bad})
    insert = ids.clone()
    insert[:, 5 + 64 + 11:5 + 64 + 11 + NE_] = 7                   # tool tokens without their [EMB] slots
    with pytest.raises(NotImplementedError):
        tr(**{**kw, "input_ids": insert.cuda()})
    m.vis_encoder.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="freeze_vis_encoder"):
        tr(**kw)
