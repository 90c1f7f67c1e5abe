"""CPU: host logic of right-padded training (visionllm_b200/train.py) -- the attention mask turned into key lengths
through the decoder's fwd+bwd (Llama against HF autograd, InternLM2 against the reference's own class via
tests/golden/train_internlm2_padded.npz, both at 1e-4), the freeze methods of the composite and the refusals of its training wrapper.  The
kernels are replaced in this test only by torch fp32 stand-ins, as in tests/test_train_logic_cpu.py."""
import os
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from test_train_internlm2_cpu import rel, stand_ins  # noqa: E402,F401
from test_train_logic_cpu import train_stand_ins  # noqa: E402,F401


def masked_attention_backward(qkv5, do, scale, seqlens=None):
    """fp32 autograd of causal (grouped-query) attention with key lengths (HF's mask: j <= i and j < len) on the packed
    [B, T, G + 2, nkv, D] rows."""
    with torch.enable_grad():
        x = qkv5.detach().float().requires_grad_(True)
        B, T, parts, nkv, D = x.shape
        G = parts - 2
        q = x[:, :, :G].flatten(2, 3)
        k = x[:, :, G].repeat_interleave(G, 2)
        v = x[:, :, G + 1].repeat_interleave(G, 2)
        s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
        i = torch.arange(T)
        lens = seqlens.long() if seqlens is not None else torch.full((B,), T)
        blocked = (i[None, :] > i[:, None])[None] | (i[None, None, :] >= lens[:, None, None])
        s = s.masked_fill(blocked[:, None], float("-inf"))
        o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v).reshape(B, T, -1)
        o.backward(do.float().reshape(B, T, -1))
    return x.grad


class _LinearF32:
    """LinearFn in fp32 (its backward stages dy in bf16 for the GEMM kernels, a 2^-9 rounding that would mask a 1e-4
    comparison; its host logic is covered by tests/test_train_logic_cpu.py)."""

    @staticmethod
    def apply(x, w, out_f32=False, residual=None, bias=None):
        y = F.linear(x.float(), w.float(), None if bias is None else bias.float())
        return y if residual is None else y + residual


@pytest.mark.parametrize("T", [77, 256])
def test_padded_decoder_matches_hf_with_the_same_mask(train_stand_ins, monkeypatch, T):
    from transformers import LlamaConfig, LlamaForCausalLM
    import visionllm_b200.train as TR
    from visionllm_b200.llama import B200LlamaForCausalLM
    monkeypatch.setattr(TR, "attention_backward_packed", masked_attention_backward)
    monkeypatch.setattr(TR, "LinearFn", _LinearF32)
    cfg = LlamaConfig(hidden_size=128, intermediate_size=352, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, vocab_size=97, rms_norm_eps=1e-5, attn_implementation="eager")
    torch.manual_seed(0)
    hf = LlamaForCausalLM(cfg).float().eval()
    g = torch.Generator().manual_seed(1)
    B = 3
    lens = torch.tensor([T, T // 2, 5])
    mask = (torch.arange(T)[None] < lens[:, None]).long()
    emb = torch.randn(B, T, 128, generator=g) * 0.5
    labels = torch.randint(0, 97, (B, T), generator=g)
    labels[mask == 0] = -100
    e = emb.clone().requires_grad_(True)
    ref = hf(inputs_embeds=e, attention_mask=mask).logits
    ref_loss = F.cross_entropy(ref[:, :-1].reshape(-1, 97), labels[:, 1:].reshape(-1), ignore_index=-100)
    ref_loss.backward()
    lm = B200LlamaForCausalLM(cfg)
    lm.load_state_dict(hf.state_dict())
    tr = TR.B200LlamaForCausalLMTrain(lm.float())
    e2 = emb.clone().requires_grad_(True)
    loss, logits, _ = tr(e2, labels, attention_mask=mask)
    loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss)) < 1e-4 * abs(float(ref_loss))
    valid = mask.bool()
    assert (logits[valid] - ref[valid]).abs().max() < 1e-4
    assert (e2.grad - e.grad).abs().max() <= 1e-4 * e.grad.abs().max() + 1e-8
    assert (e2.grad[~valid] == 0).all() and (e.grad[~valid] == 0).all()            # padded positions take no gradient
    got = dict(lm.named_parameters())
    for n, p in hf.named_parameters():
        if p.grad is not None:
            assert (got[n].grad - p.grad).abs().max() <= 1e-4 * p.grad.abs().max() + 1e-8, n
    left = mask.flip(1)                                          # left padding is not expressible as key lengths
    with pytest.raises(NotImplementedError, match="right-padded"):
        tr(emb, labels, attention_mask=left)


def test_padded_internlm2_matches_reference_golden_fp32(stand_ins, monkeypatch):
    """B200InternLM2ForCausalLMTrain with a right-padded, ragged attention_mask against the fp32 leg of
    tests/golden/train_internlm2_padded.npz (the reference's own InternLM2ForCausalLM, its own 4-D mask) at 1e-4."""
    import json
    import numpy as np
    import visionllm_b200.train as TR
    from train_internlm2_padded_inputs import WEIGHT_SEED, checksum, inputs
    from weights_util import key_shapes, seeded_state_dict
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    monkeypatch.setattr(TR, "attention_backward_packed", masked_attention_backward)
    g = np.load(os.path.join(ROOT, "tests", "golden", "train_internlm2_padded.npz"))
    cfg = SimpleNamespace(rope_scaling=None, hidden_act="silu", bias=False, pad_token_id=None, **json.loads(str(g["config"])))
    lm = B200InternLM2ForCausalLM(cfg)
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(lm)], "state-dict keys differ from the reference"
    lm.load_state_dict(seeded_state_dict(lm, WEIGHT_SEED))
    tr = TR.B200InternLM2ForCausalLMTrain(lm.float())
    emb, labels, mask = inputs()
    assert torch.equal(checksum(emb, labels), torch.from_numpy(g["inputs_checksum"])) and (mask.numpy() == g["mask"]).all()
    e = emb.clone().requires_grad_(True)
    loss, logits, _ = tr(e, labels, attention_mask=mask)
    loss.backward()
    assert abs(float(loss.detach()) - float(g["loss_f32"])) <= 1e-4 * abs(float(g["loss_f32"]))
    assert (e.grad[mask == 0] == 0).all()
    got = {"logits": logits.detach(), "d_emb": e.grad}
    got.update({"grad/" + n: p.grad for n, p in lm.named_parameters() if p.grad is not None})
    assert sorted(k[5:] for k in got if k.startswith("grad/")) == json.loads(str(g["params"]))
    for key, t in got.items():
        idx = torch.from_numpy(g[key + "/idx"]).long()
        a, r = t.detach().float().reshape(-1)[idx], torch.from_numpy(g[key + "/f32"])
        assert rel(a, r) <= 1e-4, (key, rel(a, r))


class _Tiny(nn.Module):
    def __init__(self, n=4):
        super().__init__()
        self.lin = nn.Linear(n, n)
        self.config = SimpleNamespace(hidden_size=n)


def _composite():
    from transformers import LlamaConfig
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.modeling import B200VisionLLMv2Model
    llm = B200LlamaForCausalLM(LlamaConfig(hidden_size=16, intermediate_size=32, num_hidden_layers=1, num_attention_heads=1,
                                           num_key_value_heads=1, vocab_size=50))
    cfg = SimpleNamespace(use_pixelshuffle=False, vl_bridge_type="mlp2x_gelu", num_embs=2, imp_token_id=40, emb_token_id=45,
                          det_tool_id=30, seg_tool_id=-1, grd_tool_id=-1, pose_tool_id=31)
    return B200VisionLLMv2Model(cfg, _Tiny(), llm)


def test_freeze_methods_follow_the_reference():
    m = _composite()
    m.freeze_vis_encoder()
    assert not any(p.requires_grad for p in m.vis_encoder.parameters())
    m.freeze_vl_bridge()
    assert not any(p.requires_grad for p in m.vl_bridge.parameters())
    m.freeze_emb_embeddings()
    assert not m.emb_embeddings_det.weight.requires_grad and not m.emb_embeddings_pose.weight.requires_grad
    assert all(p.requires_grad for p in m.llm.parameters())
    m.freeze_llm()
    assert not any(p.requires_grad for p in m.parameters())
    m.freeze_region_encoder()                                    # no region encoder: nothing to do


def test_training_wrapper_refusals_come_before_any_kernel():
    from visionllm_b200.train import B200VisionLLMv2ModelTrain
    tr = B200VisionLLMv2ModelTrain(_composite())
    ids = torch.randint(0, 30, (2, 8))
    for kw in (dict(targets=[{}]), dict(images_aug=[torch.zeros(3, 8, 8)]), dict(regions=[torch.ones(1, 8, 8)]),
               dict(past_key_values=((),)), dict(use_cache=True), dict(inputs_embeds=torch.zeros(2, 8, 16)), dict()):
        with pytest.raises(NotImplementedError):                 # the last: a CPU batch
            tr(input_ids=ids, **kw)
