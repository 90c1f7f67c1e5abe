"""H100-native Llama decoder (Vicuna-7B): drop-in for HF ``LlamaForCausalLM`` as the reference uses it
(visionllmv2/model/modeling_visionllmv2.py:143,420,724-738: inputs_embeds in, hidden_states[-1] and
fp32 logits out; RMSNorm := apex FusedRMSNorm via visionllmv2/train/llama_forward_monkey_patch.py:168-180).

State-dict names are HF's (model.embed_tokens, model.layers.N.self_attn.{q,k,v,o}_proj,
mlp.{gate,up,down}_proj, input_layernorm, post_attention_layernorm, model.norm, lm_head).  At first
forward the q/k/v weights are packed into one [3H, H] operand and gate/up are row-interleaved so SwiGLU
runs in the GEMM epilogue.  Per layer: RMSNorm, QKV GEMM, RoPE (q and k in one launch, in place),
fused causal attention, O GEMM (+residual), RMSNorm, gate|up GEMM (SwiGLU), down GEMM (+residual).
Forward only; grouped-query attention (InternLM2-style num_key_value_heads) supported.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops


class LlamaRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        return ops.rmsnorm(x, self.weight, self.variance_epsilon)


class LlamaAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        H = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.num_kv_heads = getattr(config, "num_key_value_heads", None) or self.num_heads
        self.head_dim = getattr(config, "head_dim", None) or H // self.num_heads
        bias = bool(getattr(config, "attention_bias", False))
        self.q_proj = nn.Linear(H, self.num_heads * self.head_dim, bias=bias)
        self.k_proj = nn.Linear(H, self.num_kv_heads * self.head_dim, bias=bias)
        self.v_proj = nn.Linear(H, self.num_kv_heads * self.head_dim, bias=bias)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, H, bias=bias)
        self._packed = None

    def packed_qkv(self):
        ws = (self.q_proj.weight, self.k_proj.weight, self.v_proj.weight)
        key = tuple((w.data_ptr(), w._version) for w in ws)
        if self._packed is None or self._packed[0] != key:
            w = torch.cat([x.detach() for x in ws], 0).contiguous()
            b = None
            if self.q_proj.bias is not None:
                b = torch.cat([self.q_proj.bias, self.k_proj.bias, self.v_proj.bias]).detach().contiguous()
            self._packed = (key, w, b)
        return self._packed[1], self._packed[2]


class LlamaMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        H, I = config.hidden_size, config.intermediate_size
        if getattr(config, "hidden_act", "silu") != "silu":
            raise NotImplementedError("LlamaMLP: only SwiGLU (hidden_act='silu')")
        self.gate_proj = nn.Linear(H, I, bias=False)
        self.up_proj = nn.Linear(H, I, bias=False)
        self.down_proj = nn.Linear(I, H, bias=False)
        self._packed = None

    def packed_gate_up(self):
        g, u = self.gate_proj.weight, self.up_proj.weight
        key = (g.data_ptr(), g._version, u.data_ptr(), u._version)
        if self._packed is None or self._packed[0] != key:
            w = torch.stack([g.detach(), u.detach()], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous()
            self._packed = (key, w)
        return self._packed[1]


def decoder_layer_forward(x, cos, sin, seqlens, norm1_w, norm2_w, eps, wqkv, bqkv, wo, bo, w_gate_up, w_down,
                          nq, nkv, D):
    """One pre-norm decoder layer on packed operands (shared by the Llama and InternLM2 drop-ins): RMSNorm, packed
    QKV GEMM, in-place RoPE on the q and k heads, fused causal attention (GQA aware), O GEMM (+residual), RMSNorm,
    gate|up GEMM with SwiGLU epilogue, down GEMM (+residual)."""
    B, T, H = x.shape
    qkv = ops.linear(ops.rmsnorm(x, norm1_w, eps), wqkv, bias=bqkv)          # [B, T, (nq + 2 nkv) D]
    ops.rope_(qkv.view(B * T, (nq + 2 * nkv) * D), cos, sin, nq + nkv, D)
    q = qkv[..., :nq * D].unflatten(-1, (nq, D))
    k = qkv[..., nq * D:(nq + nkv) * D].unflatten(-1, (nkv, D))
    v = qkv[..., (nq + nkv) * D:].unflatten(-1, (nkv, D))
    ctx = ops.attention(q, k, v, causal=True, seqlens=seqlens)
    x = ops.linear(ctx, wo, bias=bo, residual=x)
    h = ops.linear(ops.rmsnorm(x, norm2_w, eps), w_gate_up, act="swiglu")
    return ops.linear(h, w_down, residual=x)


def rope_tables(position_ids, head_dim, theta, dtype):
    """cos/sin [B*T, D] in the model dtype: fp32 angles then cast, like HF LlamaRotaryEmbedding and
    InternLM2RotaryEmbedding (internlm2/modeling_internlm2.py:132-166)."""
    dev = position_ids.device
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64, device=dev).float() / head_dim))
    fr = position_ids.reshape(-1, 1).float() * inv[None, :]
    emb = torch.cat((fr, fr), -1)
    return emb.cos().to(dtype).contiguous(), emb.sin().to(dtype).contiguous()


def right_padding_lengths(attention_mask):
    """attention_mask [B, T] (1 = real) -> int32 key lengths, or None when nothing is padded.  Only right padding
    is expressible as lengths (the reference tokenizer pads right, train.py:345)."""
    if attention_mask is None or bool(attention_mask.all()):
        return None
    am = attention_mask.to(torch.int32)
    lens = am.sum(-1).to(torch.int32)
    T = am.shape[1]
    if not bool((am == (torch.arange(T, device=am.device)[None] < lens[:, None]).int()).all()):
        raise NotImplementedError("attention_mask must be right-padded")
    return lens


class LlamaDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self_attn = LlamaAttention(config)
        self.mlp = LlamaMLP(config)
        self.input_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, x, cos, sin, seqlens=None):
        at = self.self_attn
        wqkv, bqkv = at.packed_qkv()
        return decoder_layer_forward(x, cos, sin, seqlens, self.input_layernorm.weight,
                                     self.post_attention_layernorm.weight, self.input_layernorm.variance_epsilon,
                                     wqkv, bqkv, at.o_proj.weight, at.o_proj.bias, self.mlp.packed_gate_up(),
                                     self.mlp.down_proj.weight, at.num_heads, at.num_kv_heads, at.head_dim)


class LlamaModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size)
        self.layers = nn.ModuleList([LlamaDecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self._rope = None

    def rope_tables(self, position_ids, dtype):
        cfg = self.config
        D = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
        theta = getattr(cfg, "rope_theta", None)
        if theta is None:
            rp = getattr(cfg, "rope_parameters", None) or {}
            theta = rp.get("rope_theta", 10000.0) if isinstance(rp, dict) else 10000.0
        return rope_tables(position_ids, D, theta, dtype)

    @torch.no_grad()
    def forward(self, inputs_embeds, attention_mask=None, position_ids=None, output_hidden_states=False):
        B, T, _ = inputs_embeds.shape
        dev = inputs_embeds.device
        seqlens = right_padding_lengths(attention_mask)
        if position_ids is None:
            position_ids = torch.arange(T, device=dev)[None].expand(B, T)
        cos, sin = self.rope_tables(position_ids, inputs_embeds.dtype)
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


class B200LlamaForCausalLM(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = LlamaModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)

    @property
    def dtype(self):
        return self.lm_head.weight.dtype

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, use_cache=False, output_attentions=False, output_hidden_states=False,
                return_dict=True, compute_logits=True, logits_rows=None):
        if past_key_values is not None or use_cache:
            raise NotImplementedError("KV-cache decoding is outside the forward hot path (SURVEY 3.4)")
        if inputs_embeds is None:
            inputs_embeds = self.model.embed_tokens(input_ids)
        out = self.model(inputs_embeds, attention_mask, position_ids, output_hidden_states)
        logits = None
        if logits_rows is not None:
            # lm_head on the requested rows only (SURVEY 8f rank 2): logits_rows int64 [n] indexes the flattened [B*T]
            # positions (negative = from the end); returns fp32 [n, V].  The all-positions form below stays the default
            # (what mv2.py:733-738 computes); eval loops that only read a few rows skip a ~400 MB fp32 write per batch.
            B, T, H = out.last_hidden_state.shape
            V = self.config.vocab_size
            Vp = (V + 3) // 4 * 4
            rows = ops.gather_rows(out.last_hidden_state.view(B * T, H), logits_rows.to(torch.int64).contiguous())
            buf = torch.empty((rows.shape[0], Vp), dtype=torch.float32, device=rows.device)
            ops.linear(rows, self.lm_head.weight, out=buf[:, :V])
            logits = buf[:, :V]
        elif compute_logits:
            # fp32 logits for every position, like `logits = self.llm.lm_head(hidden); logits.float()` (mv2.py:733-738);
            # the fp32 convert is the GEMM's store format, not a second pass.  Row pitch padded to 16 bytes.
            B, T, H = out.last_hidden_state.shape
            V = self.config.vocab_size
            Vp = (V + 3) // 4 * 4
            buf = torch.empty((B * T, Vp), dtype=torch.float32, device=inputs_embeds.device)
            ops.linear(out.last_hidden_state.view(B * T, H), self.lm_head.weight, out=buf[:, :V])
            logits = buf[:, :V].view(B, T, V)
        return SimpleNamespace(logits=logits, hidden_states=out.hidden_states, last_hidden_state=out.last_hidden_state,
                               past_key_values=None, attentions=None)
