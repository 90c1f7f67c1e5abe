"""H100-native InternLM2 decoder (the 26B preset's LLM): drop-in for the vendored
visionllmv2/model/internlm2/modeling_internlm2.py `InternLM2ForCausalLM` as the reference calls it
(modeling_visionllmv2.py:724-736: `self.llm(inputs_embeds=..., output_hidden_states=True)`, logits through
`self.llm.output`).  State-dict names are the reference's: model.tok_embeddings, model.layers.N.attention.{wqkv,wo},
feed_forward.{w1,w2,w3}, attention_norm, ffn_norm, model.norm, output.

The reference's fused `wqkv` interleaves, per KV head, (q_per_kv query heads, k, v) along the output rows
(:337-349); the rows are permuted once into [all q heads | all k heads | all v heads] so the packed-QKV GEMM + RoPE +
GQA attention path of llama.py applies unchanged; w1 (gate) and w3 (up) are row-interleaved for the SwiGLU epilogue
(`w2(silu(w1 x) * w3 x)`, :246).  Forward only.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .llama import decoder_layer_forward, right_padding_lengths, rope_tables


class InternLM2RMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        return ops.rmsnorm(x, self.weight, self.variance_epsilon)


class InternLM2Attention(nn.Module):
    def __init__(self, config):
        super().__init__()
        H = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.num_key_value_heads = getattr(config, "num_key_value_heads", None) or self.num_heads
        self.head_dim = H // self.num_heads
        bias = bool(getattr(config, "bias", False))
        self.wqkv = nn.Linear(H, (self.num_heads + 2 * self.num_key_value_heads) * self.head_dim, bias=bias)
        self.wo = nn.Linear(self.num_heads * self.head_dim, H, bias=bias)
        self._packed = None

    def packed_qkv(self):
        w = self.wqkv.weight
        key = (w.data_ptr(), w._version)
        if self._packed is None or self._packed[0] != key:
            nq, nkv, D = self.num_heads, self.num_key_value_heads, self.head_dim
            G = nq // nkv
            idx = torch.arange((nq + 2 * nkv) * D, device=w.device).view(nkv, G + 2, D)
            perm = torch.cat([idx[:, :G].reshape(-1), idx[:, G].reshape(-1), idx[:, G + 1].reshape(-1)])
            wq = w.detach()[perm].contiguous()
            bq = self.wqkv.bias.detach()[perm].contiguous() if self.wqkv.bias is not None else None
            self._packed = (key, wq, bq)
        return self._packed[1], self._packed[2]


class InternLM2MLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        if getattr(config, "hidden_act", "silu") != "silu":
            raise NotImplementedError("InternLM2MLP: only hidden_act='silu'")
        self.w1 = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)
        self.w3 = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)
        self.w2 = nn.Linear(config.intermediate_size, config.hidden_size, bias=False)
        self._packed = None

    def packed_gate_up(self):
        g, u = self.w1.weight, self.w3.weight
        key = (g.data_ptr(), g._version, u.data_ptr(), u._version)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, torch.stack([g.detach(), u.detach()], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous())
        return self._packed[1]


class InternLM2DecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.attention = InternLM2Attention(config)
        self.feed_forward = InternLM2MLP(config)
        self.attention_norm = InternLM2RMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.ffn_norm = InternLM2RMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, x, cos, sin, seqlens=None):
        at = self.attention
        wqkv, bqkv = at.packed_qkv()
        return decoder_layer_forward(x, cos, sin, seqlens, self.attention_norm.weight, self.ffn_norm.weight,
                                     self.attention_norm.variance_epsilon, wqkv, bqkv, at.wo.weight, at.wo.bias,
                                     self.feed_forward.packed_gate_up(), self.feed_forward.w2.weight,
                                     at.num_heads, at.num_key_value_heads, at.head_dim)


class InternLM2Model(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.tok_embeddings = nn.Embedding(config.vocab_size, config.hidden_size, getattr(config, "pad_token_id", None))
        self.layers = nn.ModuleList([InternLM2DecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = InternLM2RMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    @torch.no_grad()
    def forward(self, inputs_embeds, attention_mask=None, position_ids=None, output_hidden_states=False):
        if getattr(self.config, "rope_scaling", None) is not None:
            raise NotImplementedError("InternLM2 rope_scaling (linear / dynamic NTK) is not on the reference's path")
        B, T, _ = inputs_embeds.shape
        seqlens = right_padding_lengths(attention_mask)
        if position_ids is None:
            position_ids = torch.arange(T, device=inputs_embeds.device)[None].expand(B, T)
        D = self.config.hidden_size // self.config.num_attention_heads
        cos, sin = rope_tables(position_ids, D, getattr(self.config, "rope_theta", 10000.0), inputs_embeds.dtype)
        states = () if output_hidden_states else None
        x = inputs_embeds.contiguous()
        for layer in self.layers:
            if output_hidden_states:
                states = states + (x,)
            x = layer(x, cos, sin, seqlens)
        x = self.norm(x)
        if output_hidden_states:
            states = states + (x,)
        return SimpleNamespace(last_hidden_state=x, hidden_states=states)


class B200InternLM2ForCausalLM(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = InternLM2Model(config)
        self.output = nn.Linear(config.hidden_size, config.vocab_size, bias=False)

    @property
    def dtype(self):
        return self.output.weight.dtype

    def get_input_embeddings(self):
        return self.model.tok_embeddings

    def get_output_embeddings(self):
        return self.output

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, use_cache=False, output_attentions=False, output_hidden_states=False,
                return_dict=True, compute_logits=True):
        if past_key_values is not None or use_cache:
            raise NotImplementedError("KV-cache decoding is outside the forward hot path (SURVEY 3.4)")
        if inputs_embeds is None:
            inputs_embeds = self.model.tok_embeddings(input_ids)
        out = self.model(inputs_embeds, attention_mask, position_ids, output_hidden_states)
        logits = None
        if compute_logits:
            B, T, H = out.last_hidden_state.shape
            V = self.config.vocab_size
            Vp = (V + 3) // 4 * 4
            buf = torch.empty((B * T, Vp), dtype=torch.float32, device=inputs_embeds.device)
            ops.linear(out.last_hidden_state.view(B * T, H), self.output.weight, out=buf[:, :V])
            logits = buf[:, :V].view(B, T, V)
        return SimpleNamespace(logits=logits, hidden_states=out.hidden_states, last_hidden_state=out.last_hidden_state,
                               past_key_values=None, attentions=None)
