"""H100-native CLIP vision tower (the released-7B preset's encoder, SURVEY 8a-a6): drop-in for HF
``CLIPVisionModel`` as the reference calls it (visionllmv2/model/modeling_visionllmv2.py:135,565-571:
``vis_encoder(x, output_hidden_states=True).hidden_states[-2][:, 1:]``).  The arithmetic lives in third-party
transformers (pinned 4.34.0, not vendored); parity is checked against the installed ``CLIPVisionModel``.

State-dict names are HF's (vision_model.embeddings.*, vision_model.pre_layrnorm [sic], encoder.layers.N.
{self_attn.{q,k,v,out}_proj, layer_norm1, mlp.fc1, mlp.fc2, layer_norm2}, post_layernorm).  Per layer:
LayerNorm -> packed QKV GEMM (+bias) -> fused attention (d=64) -> out GEMM (+bias, +residual) -> LayerNorm ->
fc1 GEMM (+bias, quick-GELU epilogue) -> fc2 GEMM (+bias, +residual).  Forward only.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops


class _LN(nn.LayerNorm):
    def forward(self, x):
        return ops.layernorm(x, self.weight, self.bias, self.eps)


class CLIPVisionEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embed_dim, self.patch_size = config.hidden_size, config.patch_size
        self.class_embedding = nn.Parameter(torch.randn(self.embed_dim))
        self.patch_embedding = nn.Conv2d(config.num_channels, self.embed_dim, self.patch_size, self.patch_size,
                                         bias=False)
        self.num_positions = (config.image_size // config.patch_size) ** 2 + 1
        self.position_embedding = nn.Embedding(self.num_positions, self.embed_dim)
        self._w2d = None

    def forward(self, pixel_values):
        n, c, H, W = pixel_values.shape
        p = self.patch_size
        gh, gw = H // p, W // p
        w = self.patch_embedding.weight
        if self._w2d is None or self._w2d[0] != (w.data_ptr(), w._version):
            k = w[0].numel()
            kp = (k + 7) // 8 * 8
            w2 = torch.zeros((w.shape[0], kp), dtype=w.dtype, device=w.device)
            w2[:, :k] = w.reshape(w.shape[0], k)
            self._w2d = ((w.data_ptr(), w._version), w2, k, kp)
        _, w2, k, kp = self._w2d
        x = pixel_values.to(w2.dtype)
        cols = torch.zeros((n * gh * gw, kp), dtype=w2.dtype, device=x.device)
        cols[:, :k] = x.reshape(n, c, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(n * gh * gw, k)
        patch = ops.linear(cols, w2).view(n, gh * gw, self.embed_dim)
        cls = self.class_embedding.expand(n, 1, -1).to(patch.dtype)
        return torch.cat([cls, patch], 1) + self.position_embedding.weight.to(patch.dtype)


class CLIPAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        E = config.hidden_size
        self.num_heads, self.head_dim = config.num_attention_heads, E // config.num_attention_heads
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(E, E) for _ in range(4))
        self._packed = None

    def packed(self):
        ps = (self.q_proj, self.k_proj, self.v_proj)
        key = tuple((m.weight.data_ptr(), m.weight._version, m.bias._version) for m in ps)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, torch.cat([m.weight.detach() for m in ps], 0).contiguous(),
                            torch.cat([m.bias.detach() for m in ps], 0).contiguous())
        return self._packed[1], self._packed[2]


class CLIPEncoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        E = config.hidden_size
        self.self_attn = CLIPAttention(config)
        self.layer_norm1 = _LN(E, eps=config.layer_norm_eps)
        self.mlp = nn.Module()
        self.mlp.fc1 = nn.Linear(E, config.intermediate_size)
        self.mlp.fc2 = nn.Linear(config.intermediate_size, E)
        self.layer_norm2 = _LN(E, eps=config.layer_norm_eps)
        act = getattr(config, "hidden_act", "quick_gelu")
        if act not in ("quick_gelu", "gelu"):
            raise NotImplementedError(f"CLIP hidden_act={act}")
        self.act = act

    def forward(self, x):
        B, N, E = x.shape
        at = self.self_attn
        w, b = at.packed()
        qkv = ops.linear(self.layer_norm1(x), w, bias=b).view(B, N, 3, at.num_heads, at.head_dim)
        ctx = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False)
        x = ops.linear(ctx, at.out_proj.weight, bias=at.out_proj.bias, residual=x)
        h = ops.linear(self.layer_norm2(x), self.mlp.fc1.weight, bias=self.mlp.fc1.bias, act=self.act)
        return ops.linear(h, self.mlp.fc2.weight, bias=self.mlp.fc2.bias, residual=x)


class CLIPVisionTransformer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embeddings = CLIPVisionEmbeddings(config)
        self.pre_layrnorm = _LN(config.hidden_size, eps=config.layer_norm_eps)      # HF's spelling
        self.encoder = nn.Module()
        self.encoder.layers = nn.ModuleList([CLIPEncoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.post_layernorm = _LN(config.hidden_size, eps=config.layer_norm_eps)


class B200CLIPVisionModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.vision_model = CLIPVisionTransformer(config)

    @property
    def dtype(self):
        return self.vision_model.post_layernorm.weight.dtype

    @torch.no_grad()
    def forward(self, pixel_values=None, output_attentions=None, output_hidden_states=None, return_dict=None):
        vm = self.vision_model
        x = vm.pre_layrnorm(vm.embeddings(pixel_values))
        states = () if output_hidden_states else None
        for layer in vm.encoder.layers:
            if output_hidden_states:
                states = states + (x,)
            x = layer(x)
        if output_hidden_states:
            states = states + (x,)
        pooled = vm.post_layernorm(x[:, 0, :].contiguous())
        return SimpleNamespace(last_hidden_state=x, pooler_output=pooled, hidden_states=states, attentions=None)
