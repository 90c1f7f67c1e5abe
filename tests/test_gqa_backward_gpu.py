"""GPU: grouped-query attention backward (visionllm_b200/train.py) and what it is built from -- the grouped batched GEMM
(vllm_gemm_bf16_batched_grouped, csrc/gemm.cu) and the grouped head stacking (vllm_head_stack_qkv_bf16,
csrc/train_ops.cu).

  - GEMM bit-identities: group = 1 is vllm_gemm_bf16_batched (every causal mode, both tile widths); broadcast is the
    batched GEMM on K / V repeated G times; reduce is one gemm_tn per KV head over the concatenated G*T axis with the
    causal region zero-filled (equal up to the sign of zero: a skipped k-block of zeros adds +0 to the accumulator).
  - GEMM fp64 bound: |out - ref| <= E + one output rounding, E = ceil(K_total / 16) * 2^-24 * (|A| @ |B|^T) (the form
    of tests/test_gemm_epilogue_gpu.py), no max|ref| term.
  - Memory: outputs are views inside NaN / sentinel buffers; every element is written, nothing outside changes, and
    every documented rejection returns its code with C untouched.
  - Head stacking == torch slicing / permute, bit for bit, with NaN in the pitch gap; the round trip is exact.
  - Attention backward vs fp32 autograd with repeat_kv (the bound of test_train_gpu.py's MHA test).
  - Decoders: B200LlamaForCausalLMTrain with num_key_value_heads < num_attention_heads against HF LlamaForCausalLM
    autograd, and B200InternLM2ForCausalLMTrain against tests/golden/train_internlm2_small.npz (the reference's own
    InternLM2ForCausalLM under autograd), both under the module rule of test_decoder_fwd_bwd_matches_hf_autograd:
        rel_l2(ours, ref_fp32) <= 2 * rel_l2(ref_bf16, ref_fp32) + 3e-3   (gradients; 1.5x + 1e-3 for loss / logits).
"""
import json
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from visionllm_b200 import _lib  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILES = {"1": _lib.GEMM_DEFAULT, "2": _lib.GEMM_WIDE_TILE}     # tile width in 128-column units
SENTINEL = 4320.0                                              # exact in bf16 and fp32; the kernel never writes it here
EINVAL, EUNSUPPORTED = -1, -2


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def rel(a, b):
    return float(torch.linalg.norm(a.float() - b.float()) / (torch.linalg.norm(b.float()) + 1e-30))


def stream():
    return torch.cuda.current_stream().cuda_stream


def grouped(A, B, C, n_batch, group, reduce, M, N, K, causal, a_mn, b_mn):
    """vllm_gemm_bf16_batched_grouped into C (a view); returns the code."""
    return _lib.lib().vllm_gemm_bf16_batched_grouped(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0),
                                                     int(b_mn), C.data_ptr(), C.stride(0), n_batch, group, int(reduce), M, N,
                                                     K, causal, 1 if C.dtype == torch.float32 else 0, stream())


def batched(A, B, C, n_batch, M, N, K, causal, a_mn, b_mn):
    return _lib.lib().vllm_gemm_bf16_batched(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0), int(b_mn),
                                             C.data_ptr(), C.stride(0), n_batch, M, N, K, causal,
                                             1 if C.dtype == torch.float32 else 0, stream())


def boxed(rows, cols, dtype, fill=float("nan")):
    """A [rows + 2, ld] sentinel buffer (ld > cols, 16-byte pitch) and its [rows, cols] view at row 1, filled with `fill`."""
    per16 = 16 // torch.tensor([], dtype=dtype).element_size()
    ld = (cols + per16) // per16 * per16
    buf = torch.full((rows + 2, ld), SENTINEL, dtype=dtype, device="cuda")
    view = buf[1:rows + 1, :cols]
    view.fill_(fill)
    return buf, view


def outside_untouched(buf, rows, cols):
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    mask[1:rows + 1, :cols] = False
    return bool((buf[mask] == SENTINEL).all())


def rand(rows, cols, g, scale=1.0):
    return (torch.randn(rows, cols, device="cuda", generator=g) * scale).bfloat16()


def causal_probs(n, T, g):
    """n stacked [T, T] bf16 matrices, zero above the diagonal (a causal P / dS)."""
    return (torch.randn(n, T, T, device="cuda", generator=g) * 0.3).bfloat16().tril().view(n * T, T)


# the three operand forms of the attention backward: (a_mn, b_mn, A rows per matrix, B rows per matrix, N, K)
def forms(T, D):
    return {"qk": (0, 0, T, T, T, D),          # S = Q K^T, dP = dO V^T:  A [T, D], B [T, D] K-major, N = T, K = D
            "pdo": (1, 1, T, T, D, T),         # dV = P^T dO, dK = dS^T Q: A [T(k), T(m)], B [T(k), D] MN-major, K = T
            "dsk": (0, 1, T, T, D, T)}         # dQ = dS K: A [T, T] K-major, B [T(k), D] MN-major


def operands_for(form, n_a, n_b, T, D, g):
    a_mn, b_mn, _, _, N, K = forms(T, D)[form]
    A = rand(n_a * T, D, g) if form == "qk" else causal_probs(n_a, T, g)
    B = rand(n_b * T, D, g)
    return A, B, a_mn, b_mn, N, K


# ---------------------------------------------------------------------------------------------------------------------
# 1. bit-identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tile", list(TILES))
@pytest.mark.parametrize("causal,form", [(0, "qk"), (1, "qk"), (0, "pdo"), (2, "pdo"), (0, "dsk"), (3, "dsk")])
def test_group_one_is_the_batched_gemm(causal, form, tile):
    T, D, n = 512, 128, 3
    g = torch.Generator(device="cuda").manual_seed(100 + causal)
    A, B, a_mn, b_mn, N, K = operands_for(form, n, n, T, D, g)
    with _lib.knob("gemm_set_variant", TILES[tile]):
        for dt in (torch.bfloat16, torch.float32):
            c1 = torch.full((n * T, N), SENTINEL, dtype=dt, device="cuda")
            c2 = c1.clone()
            assert grouped(A, B, c1, n, 1, 0, T, N, K, causal, a_mn, b_mn) == 0
            assert batched(A, B, c2, n, T, N, K, causal, a_mn, b_mn) == 0
            assert same_bits(c1, c2), (dt, "group = 1 differs from vllm_gemm_bf16_batched")


@pytest.mark.parametrize("G", [2, 4, 6, 8])
@pytest.mark.parametrize("causal,form", [(0, "qk"), (1, "qk"), (3, "dsk")])
def test_broadcast_is_the_batched_gemm_on_repeated_kv(causal, form, G):
    T, D, nkv = 256, 128, 2
    n = G * nkv
    g = torch.Generator(device="cuda").manual_seed(200 + G)
    A, B, a_mn, b_mn, N, K = operands_for(form, n, nkv, T, D, g)
    B_rep = B.view(nkv, T, D).repeat_interleave(G, 0).reshape(n * T, D)      # KV matrix j serves query matrices jG .. jG+G-1
    for tile in TILES.values():
        with _lib.knob("gemm_set_variant", tile):
            c1 = torch.full((n * T, N), SENTINEL, dtype=torch.bfloat16, device="cuda")
            c2 = c1.clone()
            assert grouped(A, B, c1, n, G, 0, T, N, K, causal, a_mn, b_mn) == 0
            assert batched(A, B_rep, c2, n, T, N, K, causal, a_mn, b_mn) == 0
            assert same_bits(c1, c2)


@pytest.mark.parametrize("G", [1, 2, 6, 8])
@pytest.mark.parametrize("causal", [0, 2])
def test_reduce_is_one_gemm_tn_over_the_group(causal, G):
    from visionllm_b200 import ops
    T, D, nkv = 256, 64, 2
    n = G * nkv
    g = torch.Generator(device="cuda").manual_seed(300 + G)
    P = causal_probs(n, T, g)                    # zero above the diagonal: the K range causal 2 skips holds zeros
    dO = rand(n * T, D, g)
    for dt in (torch.bfloat16, torch.float32):
        for tile in TILES.values():
            with _lib.knob("gemm_set_variant", tile):
                c = torch.full((nkv * T, D), SENTINEL, dtype=dt, device="cuda")
                assert grouped(P, dO, c, n, G, 1, T, D, T, causal, 1, 1) == 0
                for j in range(nkv):
                    rows = slice(j * G * T, (j + 1) * G * T)        # the G matrices of KV head j: one K axis of G*T rows
                    ref = ops.gemm_tn(P[rows], dO[rows], a_mn=True, b_mn=True, out_dtype=dt)
                    got = c[j * T:(j + 1) * T]
                    assert bool((got == ref).all()), (dt, j, "reduce != gemm_tn over the group's G*T rows")


# ---------------------------------------------------------------------------------------------------------------------
# 2. fp64 bound and memory
# ---------------------------------------------------------------------------------------------------------------------
def dense(A, B, a_mn, b_mn, n_a, n_b, T, D):
    """fp64 per-matrix A_i and B_i as [M, K] / [N, K] stacks."""
    Ad = A.double().view(n_a, -1, A.shape[1])
    Bd = B.double().view(n_b, -1, B.shape[1])
    return (Ad.transpose(1, 2) if a_mn else Ad), (Bd.transpose(1, 2) if b_mn else Bd)


@pytest.mark.parametrize("case", ["S_g6_c1", "dQ_g6_c3", "dV_g6_c2", "dV_g4_c0", "S_g2_c0"])
def test_grouped_gemm_fp64_bound_and_memory(case):
    T, D, nkv = 256, 128, 2
    kind, G, causal = case.split("_")[0], int(case.split("_")[1][1:]), int(case.split("_")[2][1:])
    n = G * nkv
    g = torch.Generator(device="cuda").manual_seed(400 + G + causal)
    form = {"S": "qk", "dQ": "dsk", "dV": "pdo"}[kind]
    reduce = kind == "dV"
    A, B, a_mn, b_mn, N, K = operands_for(form, n, n if reduce else nkv, T, D, g)
    Ad, Bd = dense(A, B, a_mn, b_mn, n, n if reduce else nkv, T, D)
    if reduce:                                   # output j: the G products of its group on one K axis of G*T
        Ad = Ad.view(nkv, G, T, T).permute(0, 2, 1, 3).reshape(nkv, T, G * T)
        Bd = Bd.view(nkv, G, D, T).permute(0, 2, 1, 3).reshape(nkv, D, G * T)
        K_total = G * T
    else:
        Bd = Bd.repeat_interleave(G, 0)
        K_total = K
    ref = Ad @ Bd.transpose(1, 2)
    E = math.ceil(K_total / 16) * 2.0 ** -24 * (Ad.abs() @ Bd.abs().transpose(1, 2))
    n_out = nkv if reduce else n
    valid = torch.ones(T, N, dtype=torch.bool, device="cuda")
    if causal == 1:                              # tiles strictly above the diagonal are skipped (left as they were)
        valid = torch.ones(T, T, dtype=torch.bool, device="cuda").tril()
    for dt, out_round in ((torch.float32, 2.0 ** -23), (torch.bfloat16, 2.0 ** -8)):
        buf, c = boxed(n_out * T, N, dt)
        assert grouped(A, B, c, n, G, int(reduce), T, N, K, causal, a_mn, b_mn) == 0
        assert outside_untouched(buf, n_out * T, N), (dt, "a store landed outside C")
        got = c.view(n_out, T, N)
        assert not got[:, valid].isnan().any(), (dt, "elements of C were never written")
        err = (got.double() - ref).abs()[:, valid]
        bound = (E + out_round * (ref.abs() + E))[:, valid]
        assert bool((err <= bound).all()), (dt, float((err / bound).max()))


def test_grouped_gemm_rejections_leave_c_untouched():
    T, D = 256, 64
    g = torch.Generator(device="cuda").manual_seed(500)
    P = causal_probs(4, T, g)
    X = rand(4 * T, D, g)
    Q = rand(4 * T, D, g)
    cases = [  # (what, args, expected code)
        ("group 0", (P, X, 4, 0, 1, T, D, T, 2, 1, 1), EINVAL),
        ("group < 0", (P, X, 4, -2, 0, T, D, T, 0, 1, 1), EINVAL),
        ("n_batch % group", (P, X, 4, 3, 1, T, D, T, 2, 1, 1), EINVAL),
        ("reduce not 0 / 1", (P, X, 4, 2, 2, T, D, T, 0, 1, 1), EINVAL),
        ("reduce + causal 1", (P, X, 4, 2, 1, T, D, T, 1, 1, 1), EINVAL),
        ("reduce + causal 3", (P, X, 4, 2, 1, T, D, T, 3, 1, 1), EINVAL),
        ("reduce + causal 2 with K != M", (P, X, 4, 2, 1, T, D, 192, 2, 1, 1), EINVAL),
        ("reduce, K-major A", (Q, X, 4, 2, 1, T, D, D, 0, 0, 1), EUNSUPPORTED),
        ("reduce, K-major B", (P, Q, 4, 2, 1, T, D, T, 0, 1, 0), EUNSUPPORTED),
        ("M % 256", (Q, Q, 4, 2, 0, 128, 128, D, 0, 0, 0), EUNSUPPORTED),
        ("misaligned A", (Q[:, 1:], Q, 4, 2, 0, T, T, D - 8, 0, 0, 0), -3),
    ]
    for what, (A, B, nb, grp, red, M, N, K, causal, a_mn, b_mn), code in cases:
        buf, c = boxed(nb * M, max(N, 8), torch.bfloat16, fill=1.0)
        before = buf.clone()
        rc = grouped(A, B, c, nb, grp, red, M, N, K, causal, a_mn, b_mn)
        torch.cuda.synchronize()
        assert rc == code, (what, rc)
        assert same_bits(buf, before), (what, "C changed")


# ---------------------------------------------------------------------------------------------------------------------
# 3. head stacking
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq,nkv,D", [(4, 4, 64), (12, 2, 64), (8, 1, 128), (6, 2, 40)])
def test_head_stack_qkv_matches_torch_and_round_trips(nq, nkv, D):
    from visionllm_b200.train import head_stack_qkv
    B, T = 2, 37
    W = (nq + 2 * nkv) * D
    ld = W + 24                                   # a pitch gap of 24 elements, NaN
    g = torch.Generator(device="cuda").manual_seed(600 + nq)
    rows = torch.full((B, T, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    rows[..., :W] = torch.randn(B, T, W, device="cuda", generator=g).bfloat16()
    packed = rows[..., :W]
    stk = head_stack_qkv(packed, nq, nkv, D)
    q = packed[..., :nq * D].view(B, T, nq, D).permute(0, 2, 1, 3).reshape(-1, D)
    k = packed[..., nq * D:(nq + nkv) * D].view(B, T, nkv, D).permute(0, 2, 1, 3).reshape(-1, D)
    v = packed[..., (nq + nkv) * D:].view(B, T, nkv, D).permute(0, 2, 1, 3).reshape(-1, D)
    assert same_bits(stk, torch.cat([q, k, v], 0))
    back = torch.full_like(rows, float("nan"))
    head_stack_qkv(back[..., :W], nq, nkv, D, stacks=stk)
    assert same_bits(back[..., :W], packed)
    assert back[..., W:].isnan().all(), "the pitch gap was written"


# ---------------------------------------------------------------------------------------------------------------------
# 4. attention backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [256, 512])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [1, 2, 6, 8])
def test_gqa_attention_backward_matches_autograd(G, D, T):
    from visionllm_b200.train import attention_backward
    g = torch.Generator(device="cuda").manual_seed(700 + G + D + T)
    B, nkv = 2, 2 if G < 8 else 1
    nq = G * nkv
    q, do = ((torch.randn(B, T, nq, D, device="cuda", generator=g) * 0.5).bfloat16() for _ in range(2))
    k, v = ((torch.randn(B, T, nkv, D, device="cuda", generator=g) * 0.5).bfloat16() for _ in range(2))
    scale = D ** -0.5
    dq, dk, dv = attention_backward(q, k, v, do, scale)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf.repeat_interleave(G, 2)) * scale
    s = s.masked_fill(~torch.ones(T, T, device="cuda", dtype=torch.bool).tril(), float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf.repeat_interleave(G, 2))
    o.backward(do.float())
    for got, ref, name in ((dq, qf.grad, "dq"), (dk, kf.grad, "dk"), (dv, vf.grad, "dv")):
        assert got.shape == ref.shape
        assert rel(got, ref) < 1.5e-2, (name, rel(got, ref))


# ---------------------------------------------------------------------------------------------------------------------
# 5. decoders
# ---------------------------------------------------------------------------------------------------------------------
def module_rule(loss, lg, de, params):
    """test_decoder_fwd_bwd_matches_hf_autograd's rule on (loss, logits, input grad, {name: (ours, ref32, ref16)})."""
    (l, l32, l16), (lo, lg32, lg16), (d, de32, de16) = loss, lg, de
    assert abs(l - l32) <= 1.5 * abs(l16 - l32) + 1e-3 * abs(l32), (l, l32, l16)
    assert rel(lo, lg32) <= 1.5 * rel(lg16, lg32) + 1e-3, (rel(lo, lg32), rel(lg16, lg32))
    assert rel(d, de32) <= 2 * rel(de16, de32) + 3e-3, (rel(d, de32), rel(de16, de32))
    worst = []
    for n, (a_, r32, r16) in params.items():
        a, b = rel(a_, r32), rel(r16, r32)
        worst.append((a / (2 * b + 3e-3), n, a, b))
        assert a <= 2 * b + 3e-3, (n, a, b)
    print("worst grad ratio:", max(worst)[:4])


def test_llama_gqa_decoder_fwd_bwd_matches_hf_autograd():
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    cfg = LlamaConfig(hidden_size=512, intermediate_size=1376, num_hidden_layers=2, num_attention_heads=8,
                      num_key_value_heads=2, vocab_size=1000, rms_norm_eps=1e-5, max_position_embeddings=512,
                      attn_implementation="eager")
    torch.manual_seed(0)
    hf = LlamaForCausalLM(cfg)
    sd = {k: v.to(torch.bfloat16).float() for k, v in hf.state_dict().items()}
    hf.load_state_dict(sd)
    B, T = 2, 256
    gen = torch.Generator().manual_seed(3)
    emb = (torch.randn(B, T, 512, generator=gen) * 0.5).bfloat16()
    labels = torch.randint(0, 1000, (B, T), generator=gen)
    labels[:, :100] = -100

    def hf_run(dtype):
        m = hf.to("cuda", dtype).train(False)
        for p in m.parameters():
            p.grad = None
        e = emb.to("cuda", dtype).requires_grad_(True)
        out = m(inputs_embeds=e, attention_mask=torch.ones(B, T, dtype=torch.long, device="cuda"), labels=None)
        logits = out.logits.float()
        loss = F.cross_entropy(logits[:, :-1].reshape(-1, 1000), labels.cuda()[:, 1:].reshape(-1), ignore_index=-100)
        loss.backward()
        grads = {n: p.grad.detach().float().clone() for n, p in m.named_parameters() if p.grad is not None}
        return float(loss), logits.detach(), e.grad.detach().float(), grads

    l32, lg32, de32, g32 = hf_run(torch.float32)
    l16, lg16, de16, g16 = hf_run(torch.bfloat16)
    mine = B200LlamaForCausalLM(cfg)
    mine.load_state_dict(sd)
    mine = mine.to("cuda", torch.bfloat16)
    tr = B200LlamaForCausalLMTrain(mine)
    e = emb.cuda().requires_grad_(True)
    loss, logits, _ = tr(e, labels.cuda())
    loss.backward()
    params = {n: (p.grad, g32[n], g16[n]) for n, p in mine.named_parameters() if n != "model.embed_tokens.weight"}
    assert all(p[0] is not None for p in params.values())
    module_rule((float(loss), l32, l16), (logits, lg32, lg16), (e.grad, de32, de16), params)


def test_internlm2_decoder_fwd_bwd_matches_reference_golden():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from train_internlm2_inputs import WEIGHT_SEED, checksum, inputs
    from weights_util import key_shapes, seeded_state_dict
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    gz = np.load(os.path.join(ROOT, "tests", "golden", "train_internlm2_small.npz"))
    cfg = SimpleNamespace(rope_scaling=None, hidden_act="silu", bias=False, pad_token_id=None, **json.loads(str(gz["config"])))
    lm = B200InternLM2ForCausalLM(cfg)
    assert json.loads(str(gz["keys"])) == [list(k) for k in key_shapes(lm)]
    lm.load_state_dict(seeded_state_dict(lm, WEIGHT_SEED))
    lm = lm.to("cuda", torch.bfloat16)
    tr = B200InternLM2ForCausalLMTrain(lm)
    emb, labels = inputs()
    assert torch.equal(checksum(emb, labels), torch.from_numpy(gz["inputs_checksum"])), "seeded inputs differ from the golden's"
    e = emb.cuda().bfloat16().requires_grad_(True)
    loss, logits, _ = tr(e, labels.cuda())
    loss.backward()

    def sample(key, t):
        idx = torch.from_numpy(gz[key + "/idx"]).long().cuda()
        return (t.detach().float().reshape(-1)[idx], torch.from_numpy(gz[key + "/f32"]).cuda(),
                torch.from_numpy(gz[key + "/refbf16"]).cuda())

    named = dict(lm.named_parameters())
    names = json.loads(str(gz["params"]))
    assert all(named[n].grad is not None for n in names)
    params = {n: sample("grad/" + n, named[n].grad) for n in names}
    module_rule((float(loss), float(gz["loss_f32"]), float(gz["loss_refbf16"])),
                sample("logits", logits), sample("d_emb", e.grad), params)
