"""CPU: host logic of the InternLM2 training wrapper (visionllm_b200.train.B200InternLM2ForCausalLMTrain) -- the
differentiable gather of the fused, per-KV-head interleaved `wqkv` into q | k | v, the gate|up interleave, the shared
per-layer loop with grouped-query heads, rope_theta and the loss convention -- against the fp32 leg of
tests/golden/train_internlm2_small.npz (the reference's own InternLM2ForCausalLM under autograd).  The kernels are
replaced IN THIS TEST ONLY by torch fp32 stand-ins, as in tests/test_train_logic_cpu.py; a wrong `wqkv` permutation
gradient fails here without a GPU.  LinearFn is replaced too: its backward stages the incoming gradient in bf16 for the
GEMM kernels, a 2^-9 rounding that would hide nothing at this file's 1e-4 bound (its host logic is covered by
tests/test_train_logic_cpu.py)."""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from train_internlm2_inputs import WEIGHT_SEED, checksum, inputs  # noqa: E402
from weights_util import key_shapes, seeded_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "train_internlm2_small.npz")


def rel(a, b):
    return float(torch.linalg.norm(a.double() - b.double()) / (torch.linalg.norm(b.double()) + 1e-30))


def gqa_attention_backward_packed(qkv5, do, scale):
    """fp32 autograd of causal GQA attention on the packed [B, T, G + 2, nkv, D] rows (repeat_kv of HF / the reference)."""
    with torch.enable_grad():
        x = qkv5.detach().float().requires_grad_(True)
        B, T, parts, nkv, D = x.shape
        G = parts - 2
        q = x[:, :, :G].flatten(2, 3)
        k = x[:, :, G].repeat_interleave(G, 2)
        v = x[:, :, G + 1].repeat_interleave(G, 2)
        s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
        s = s.masked_fill(~torch.ones(T, T, dtype=torch.bool).tril(), float("-inf"))
        o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v).reshape(B, T, -1)
        o.backward(do.float().reshape(B, T, -1))
    return x.grad


@pytest.fixture()
def stand_ins(monkeypatch):
    import visionllm_b200.ops as ops
    import visionllm_b200.train as TR
    from oracle import torch_kernels as K

    def gemm_tn(a, b, a_mn=False, b_mn=False, out_dtype=None):
        A = a.float().t() if a_mn else a.float()
        Bm = b.float().t() if b_mn else b.float()
        return A @ Bm.t()

    def rmsnorm_bwd(x2, w, dy2, eps):
        with torch.enable_grad():
            x = x2.detach().float().requires_grad_(True)
            wf = w.detach().float().requires_grad_(True)
            (wf * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))).backward(dy2.float())
        return x.grad, wf.grad

    def swiglu_bwd(gu, dh):
        with torch.enable_grad():
            g = gu.detach().float().requires_grad_(True)
            (F.silu(g[:, 0::2]) * g[:, 1::2]).backward(dh.float())
        return g.grad

    class CE:
        @staticmethod
        def apply(logits, labels):
            return F.cross_entropy(logits, labels, ignore_index=-100)

    class Linear:
        @staticmethod
        def apply(x, w, out_f32=False, residual=None):
            y = F.linear(x.float(), w.float())
            return y if residual is None else y + residual

    for name in ("linear", "rmsnorm", "rope_", "attention"):
        monkeypatch.setattr(ops, name, getattr(K, name))
    monkeypatch.setattr(ops, "gemm_tn", gemm_tn)
    monkeypatch.setattr(TR, "rmsnorm_bwd", rmsnorm_bwd)
    monkeypatch.setattr(TR, "swiglu_fwd", lambda gu: F.silu(gu[:, 0::2].float()) * gu[:, 1::2].float())
    monkeypatch.setattr(TR, "swiglu_bwd", swiglu_bwd)
    monkeypatch.setattr(TR, "attention_backward_packed", gqa_attention_backward_packed)
    monkeypatch.setattr(TR, "CrossEntropyFn", CE)
    monkeypatch.setattr(TR, "LinearFn", Linear)


def golden_config(g):
    c = json.loads(str(g["config"]))
    return SimpleNamespace(rope_scaling=None, hidden_act="silu", bias=False, pad_token_id=None, **c)


def test_internlm2_train_wrapper_matches_reference_fp32(stand_ins):
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    g = np.load(GOLDEN)
    cfg = golden_config(g)
    lm = B200InternLM2ForCausalLM(cfg)
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(lm)], "state-dict keys differ from the reference"
    lm.load_state_dict(seeded_state_dict(lm, WEIGHT_SEED))
    lm = lm.float()
    tr = B200InternLM2ForCausalLMTrain(lm)
    emb, labels = inputs()
    assert torch.equal(checksum(emb, labels), torch.from_numpy(g["inputs_checksum"])), "seeded inputs differ from the golden's"
    for _ in range(2):                                     # twice: nothing stale is carried between steps
        for p in lm.parameters():
            p.grad = None
        e = emb.clone().requires_grad_(True)
        loss, logits, _ = tr(e, labels)
        loss.backward()
        assert abs(float(loss.detach()) - float(g["loss_f32"])) <= 1e-4 * abs(float(g["loss_f32"]))
        got = {"logits": logits.detach(), "d_emb": e.grad}
        got.update({"grad/" + n: p.grad for n, p in lm.named_parameters() if p.grad is not None})
        assert sorted(k[5:] for k in got if k.startswith("grad/")) == json.loads(str(g["params"]))
        for key, t in got.items():
            idx = torch.from_numpy(g[key + "/idx"]).long()
            a, r = t.detach().float().reshape(-1)[idx], torch.from_numpy(g[key + "/f32"])
            assert rel(a, r) <= 1e-4, (key, rel(a, r))


def test_internlm2_wqkv_gradient_lands_in_reference_order(stand_ins):
    """The gathered q | k | v rows are a pure permutation of `wqkv`: a gradient on the gathered rows comes back to the
    reference's (G query heads, k, v)-per-KV-head order."""
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    cfg = SimpleNamespace(vocab_size=64, hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=8,
                          num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=10000.0, rope_scaling=None,
                          hidden_act="silu", bias=False, pad_token_id=None)
    lm = B200InternLM2ForCausalLM(cfg).float()
    tr = B200InternLM2ForCausalLMTrain(lm)
    layer = lm.model.layers[0]
    w = layer.attention.wqkv.weight
    wqkv = tr.layer_weights(layer)[2]
    packed, _ = layer.attention.packed_qkv()                # the forward module's (non-differentiable) permutation
    assert torch.equal(wqkv.detach(), packed)
    gy = torch.randn_like(wqkv)
    wqkv.backward(gy)
    nq, nkv, D, G = 8, 2, 16, 4
    ref = torch.empty_like(w).view(nkv, G + 2, D, -1)
    q, k, v = gy[:nq * D].view(nkv, G, D, -1), gy[nq * D:(nq + nkv) * D].view(nkv, D, -1), gy[(nq + nkv) * D:].view(nkv, D, -1)
    ref[:, :G], ref[:, G], ref[:, G + 1] = q, k, v
    assert torch.equal(w.grad, ref.view_as(w))


def test_internlm2_train_wrapper_refuses_what_it_cannot_train():
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    base = dict(vocab_size=64, hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=8,
                num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=10000.0, rope_scaling=None, hidden_act="silu",
                bias=False, pad_token_id=None)
    with pytest.raises(NotImplementedError):
        B200InternLM2ForCausalLMTrain(B200InternLM2ForCausalLM(SimpleNamespace(**{**base, "bias": True})))
    with pytest.raises(NotImplementedError):
        B200InternLM2ForCausalLMTrain(B200InternLM2ForCausalLM(SimpleNamespace(**{**base, "rope_scaling": {"type": "linear",
                                                                                                        "factor": 2.0}})))
