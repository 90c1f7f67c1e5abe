"""GPU: the training-side path (visionllm_b200/train.py; BASELINE cfg 5 "fwd+bwd step") -- every backward kernel against
torch autograd of the same op in fp32, and the whole decoder fwd+bwd (loss, parameter grads, input grad) against HF
`LlamaForCausalLM` autograd (the reference's LLM is third-party transformers) with the module rule:
    rel_l2(ours, ref_fp32) <= 2 * rel_l2(ref_bf16, ref_fp32) + 3e-3   (gradients; 1.5x + 1e-3 for the loss / logits)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from visionllm_b200 import _lib  # noqa: E402


def rel(a, b):
    return float(torch.linalg.norm(a.float() - b.float()) / (torch.linalg.norm(b.float()) + 1e-30))


@pytest.mark.parametrize("variant", [pytest.param(_lib.GEMM_DEFAULT, id="1"), pytest.param(_lib.GEMM_WIDE_TILE, id="2")])   # id: tile width / 128 columns
def test_batched_gemm_forms_of_the_attention_backward(variant):
    from visionllm_b200.train import gemm_batched
    g = torch.Generator(device="cuda").manual_seed(0)
    BH, T, D = 3, 512, 128
    q, k = ((torch.randn(BH, T, D, device="cuda", generator=g) * 0.3).bfloat16() for _ in range(2))
    p = (torch.randn(BH, T, T, device="cuda", generator=g) * 0.3).bfloat16().tril()       # causal: zero above the diagonal
    with _lib.knob("gemm_set_variant", variant):
        s = gemm_batched(q.view(BH * T, D), k.view(BH * T, D), BH, T, T, D, causal=1).view(BH, T, T)
        s_full = gemm_batched(q.view(BH * T, D), k.view(BH * T, D), BH, T, T, D).view(BH, T, T)
        dv = gemm_batched(p.view(BH * T, T), q.view(BH * T, D), BH, T, D, T, a_mn=True, b_mn=True, causal=2).view(BH, T, D)
        dv_nc = gemm_batched(p.view(BH * T, T), q.view(BH * T, D), BH, T, D, T, a_mn=True, b_mn=True).view(BH, T, D)
        dq = gemm_batched(p.view(BH * T, T), k.view(BH * T, D), BH, T, D, T, b_mn=True, causal=3).view(BH, T, D)
    ref_s = q.float() @ k.float().transpose(1, 2)
    tol = lambda ref: 2.0 ** -8 * ref.abs() + 1e-3 * ref.abs().max()  # noqa: E731
    assert ((s_full.float() - ref_s).abs() <= tol(ref_s)).all()
    low = torch.ones(T, T, device="cuda", dtype=torch.bool).tril()
    assert ((s.float() - ref_s).abs() <= tol(ref_s))[:, low].all()                        # skipped tiles are don't-care
    ref_dv = p.float().transpose(1, 2) @ q.float()
    assert ((dv.float() - ref_dv).abs() <= tol(ref_dv)).all() and ((dv_nc.float() - ref_dv).abs() <= tol(ref_dv)).all()
    ref_dq = p.float() @ k.float()
    assert ((dq.float() - ref_dq).abs() <= tol(ref_dq)).all()


def test_attention_backward_matches_autograd():
    from visionllm_b200.train import attention_backward
    g = torch.Generator(device="cuda").manual_seed(1)
    B, T, H, D = 2, 512, 3, 128
    q, k, v, do = ((torch.randn(B, T, H, D, device="cuda", generator=g) * 0.5).bfloat16() for _ in range(4))
    scale = D ** -0.5
    dq, dk, dv = attention_backward(q, k, v, do, scale)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    s = s.masked_fill(~torch.ones(T, T, device="cuda", dtype=torch.bool).tril(), float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf)
    o.backward(do.float())
    for got, ref, name in ((dq, qf.grad, "dq"), (dk, kf.grad, "dk"), (dv, vf.grad, "dv")):
        assert rel(got, ref) < 1.5e-2, (name, rel(got, ref))          # bf16 scores / probabilities (HF eager bf16 class)


def test_rmsnorm_swiglu_rope_ce_backward_match_autograd():
    from visionllm_b200 import train as TR
    g = torch.Generator(device="cuda").manual_seed(2)
    rows, C = 300, 4096
    x = (torch.randn(rows, C, device="cuda", generator=g)).bfloat16()
    w = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
    dy = (torch.randn(rows, C, device="cuda", generator=g) * 0.1).bfloat16()
    dx, dw = TR.rmsnorm_bwd(x, w, dy, 1e-5)
    xf, wf = x.float().requires_grad_(True), w.float().requires_grad_(True)
    (wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))).backward(dy.float())
    assert rel(dx, xf.grad) < 5e-3 and rel(dw, wf.grad) < 5e-3
    # SwiGLU on interleaved (gate, up) columns
    I = 1376
    gu = (torch.randn(rows, 2 * I, device="cuda", generator=g)).bfloat16()
    dh = (torch.randn(rows, I, device="cuda", generator=g) * 0.1).bfloat16()
    h = TR.swiglu_fwd(gu)
    guf = gu.float().requires_grad_(True)
    href = F.silu(guf[:, 0::2]) * guf[:, 1::2]
    href.backward(dh.float())
    assert rel(h, href) < 5e-3 and rel(TR.swiglu_bwd(gu, dh), guf.grad) < 5e-3
    # CE loss + dlogits
    R, V = 64, 32026
    logits = (torch.randn(R, V, device="cuda", generator=g) * 2).float().requires_grad_(True)
    labels = torch.randint(0, V, (R,), device="cuda", generator=g)
    labels[::5] = -100
    loss = TR.CrossEntropyFn.apply(logits, labels)
    loss.backward()
    lf = logits.detach().clone().requires_grad_(True)
    ref = F.cross_entropy(lf, labels, ignore_index=-100)
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-4 * abs(float(ref))
    assert rel(logits.grad, lf.grad) < 5e-3 and (logits.grad[::5] == 0).all()
    # RoPE backward = rotation by -theta
    T_, Hh, D = 40, 4, 128
    from visionllm_b200.llama import rope_tables
    cos, sin = rope_tables(torch.arange(T_, device="cuda")[None], D, 10000.0, torch.bfloat16)
    xq = (torch.randn(T_, 3 * Hh * D, device="cuda", generator=g)).bfloat16().requires_grad_(True)
    out = TR.RopeFn.apply(xq, cos, sin, 2 * Hh, D)
    gy = (torch.randn_like(out.float()) * 0.1).bfloat16()
    out.backward(gy)
    xr = xq.detach().float().requires_grad_(True)
    v = xr[:, :2 * Hh * D].reshape(T_, 2 * Hh, D)
    c, s = cos.float()[:, None], sin.float()[:, None]
    rot = torch.cat((-v[..., D // 2:], v[..., :D // 2]), -1)
    ref_out = torch.cat(((v * c + rot * s).reshape(T_, -1), xr[:, 2 * Hh * D:]), 1)
    ref_out.backward(gy.float())
    assert rel(out, ref_out) < 5e-3 and rel(xq.grad, xr.grad) < 5e-3


def test_decoder_fwd_bwd_matches_hf_autograd():
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    cfg = LlamaConfig(hidden_size=512, intermediate_size=1376, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=1000, rms_norm_eps=1e-5, max_position_embeddings=512,
                      attn_implementation="eager")
    torch.manual_seed(0)
    hf = LlamaForCausalLM(cfg)
    sd = {k: v.to(torch.bfloat16).float() for k, v in hf.state_dict().items()}
    hf.load_state_dict(sd)
    B, T = 2, 256
    gen = torch.Generator().manual_seed(3)
    emb = (torch.randn(B, T, 512, generator=gen) * 0.5).bfloat16()
    labels = torch.randint(0, 1000, (B, T), generator=gen)
    labels[:, :100] = -100                                       # visual positions carry no language loss

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
    assert abs(float(loss) - l32) <= 1.5 * abs(l16 - l32) + 1e-3 * abs(l32), (float(loss), l32, l16)
    assert rel(logits, lg32) <= 1.5 * rel(lg16, lg32) + 1e-3
    assert rel(e.grad, de32) <= 2 * rel(de16, de32) + 3e-3, (rel(e.grad, de32), rel(de16, de32))
    worst = []
    for n, p in mine.named_parameters():
        if n == "model.embed_tokens.weight":
            continue                                             # inputs_embeds path: the table is not touched
        assert p.grad is not None, n
        a, b = rel(p.grad, g32[n]), rel(g16[n], g32[n])
        worst.append((a / (2 * b + 3e-3), n, a, b))
        assert a <= 2 * b + 3e-3, (n, a, b)
    print("worst grad ratio:", max(worst)[:4])


def test_b200_rmsnorm_module_forward_backward():
    from visionllm_b200.norm import B200RMSNorm
    m = B200RMSNorm(1024, eps=1e-5).to("cuda", torch.bfloat16)
    with torch.no_grad():
        m.weight.copy_(1 + 0.1 * torch.randn(1024))
    x = torch.randn(3, 50, 1024, device="cuda").bfloat16().requires_grad_(True)
    y = m(x)
    y.backward(torch.ones_like(y) * 0.1)
    xf, wf = x.detach().float().requires_grad_(True), m.weight.detach().float().requires_grad_(True)
    ref = wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))
    ref.backward(torch.ones_like(ref) * 0.1)
    assert rel(y, ref) < 5e-3 and rel(x.grad, xf.grad) < 5e-3 and rel(m.weight.grad, wf.grad) < 5e-3
    with torch.no_grad():
        assert torch.equal(m(x.detach()), y.detach())            # the no-grad path is the same kernel
