"""H100-native InternViT: drop-in for the reference ``InternVisionModel``.

Mirrors visionllmv2/model/internvit/modeling_intern_vit.py (class/attribute/state-dict
names identical, so reference checkpoints load with ``load_state_dict``):

  InternVisionEmbeddings  :61-90    Conv2d(3->C, k=p, s=p) as an im2col GEMM, + cls, + learned pos
  InternAttention         :93-164   qkv GEMM -> RMSNorm(q), RMSNorm(k) over the flattened C dims (in place on
                                    the packed qkv) -> fused attention -> proj GEMM
  InternMLP               :167-179  fc1 GEMM (+bias, erf-GELU epilogue) -> fc2 GEMM
  InternVisionEncoderLayer:182-210  x += ls1*attn(norm1(x)); x += ls2*mlp(norm2(x))
                                    (bias, LayerScale and residual all live in the GEMM epilogues)
  InternVisionEncoder     :213-276  returns every layer's hidden state
  InternVisionModel       :279-343

Forward only (inference); 9 kernel launches per layer, all through the C-ABI library.
"""
from dataclasses import dataclass
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops


@dataclass
class InternVisionConfig:
    """Defaults of the reference configuration_intern_vit.py:63-82 (InternViT-6B)."""
    num_channels: int = 3
    patch_size: int = 14
    image_size: int = 224
    qkv_bias: bool = False
    hidden_size: int = 3200
    num_attention_heads: int = 25
    intermediate_size: int = 12800
    qk_normalization: bool = True
    num_hidden_layers: int = 48
    use_flash_attn: bool = True
    hidden_act: str = "gelu"
    layer_norm_eps: float = 1e-6
    dropout: float = 0.0
    drop_path_rate: float = 0.0
    attention_dropout: float = 0.0
    initializer_range: float = 0.02
    initializer_factor: float = 0.1
    output_hidden_states: bool = False
    use_return_dict: bool = True


class InternRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x, out=None):
        return ops.rmsnorm(x, self.weight, self.variance_epsilon, out=out)


class InternVisionEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embed_dim = config.hidden_size
        self.image_size = config.image_size
        self.patch_size = config.patch_size
        self.class_embedding = nn.Parameter(torch.randn(1, 1, self.embed_dim))
        self.patch_embedding = nn.Conv2d(3, self.embed_dim, kernel_size=self.patch_size, stride=self.patch_size)
        self.num_patches = (self.image_size // self.patch_size) ** 2
        self.num_positions = self.num_patches + 1
        self.position_embedding = nn.Parameter(torch.randn(1, self.num_positions, self.embed_dim))
        self._w2d = None

    def _weight_2d(self):
        # Conv2d weight [C, 3, p, p] -> K-major GEMM operand [C, Kp], K = 3*p*p padded to a multiple of 8
        w = self.patch_embedding.weight
        if self._w2d is None or self._w2d[0] is not w or self._w2d[1] != w._version:
            k = w[0].numel()
            kp = (k + 7) // 8 * 8
            w2 = torch.zeros((w.shape[0], kp), dtype=w.dtype, device=w.device)
            w2[:, :k] = w.reshape(w.shape[0], k)
            self._w2d = (w, w._version, w2, k, kp)
        return self._w2d[2], self._w2d[3], self._w2d[4]

    def forward(self, pixel_values):
        n, c, H, W = pixel_values.shape
        p = self.patch_size
        gh, gw = H // p, W // p
        w2, k, kp = self._weight_2d()
        x = pixel_values.to(w2.dtype)[:, :, :gh * p, :gw * p]
        # im2col (pure data movement): [n, c, gh, p, gw, p] -> [n*gh*gw, c*p*p]
        cols = torch.zeros((n * gh * gw, kp), dtype=w2.dtype, device=x.device)
        cols[:, :k] = x.reshape(n, c, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(n * gh * gw, k)
        patch = ops.linear(cols, w2, bias=self.patch_embedding.bias).view(n, gh * gw, self.embed_dim)
        cls = self.class_embedding.expand(n, 1, -1).to(patch.dtype)
        return torch.cat([cls, patch], dim=1) + self.position_embedding.to(patch.dtype)


class InternAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embed_dim = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = self.embed_dim // self.num_heads
        if self.head_dim * self.num_heads != self.embed_dim:
            raise ValueError("embed_dim must be divisible by num_heads")
        self.scale = self.head_dim ** -0.5
        self.qkv = nn.Linear(self.embed_dim, 3 * self.embed_dim, bias=config.qkv_bias)
        self.qk_normalization = config.qk_normalization
        if self.qk_normalization:
            self.q_norm = InternRMSNorm(self.embed_dim, eps=config.layer_norm_eps)
            self.k_norm = InternRMSNorm(self.embed_dim, eps=config.layer_norm_eps)
        self.proj = nn.Linear(self.embed_dim, self.embed_dim)

    def forward(self, x, colscale=None, residual=None):
        B, N, C = x.shape
        qkv = ops.linear(x, self.qkv.weight, bias=self.qkv.bias)          # [B, N, 3C] packed
        flat = qkv.view(B * N, 3 * C)
        if self.qk_normalization:                                          # :149-153, in place, no stack copy
            q2, k2 = flat[:, :C], flat[:, C:2 * C]
            self.q_norm(q2, out=q2)
            self.k_norm(k2, out=k2)
        v5 = qkv.view(B, N, 3, self.num_heads, self.head_dim)
        ctx = ops.attention(v5[:, :, 0], v5[:, :, 1], v5[:, :, 2], causal=False, scale=self.scale)
        return ops.linear(ctx, self.proj.weight, bias=self.proj.bias, colscale=colscale, residual=residual)


class InternMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        if config.hidden_act != "gelu":
            raise NotImplementedError("InternMLP: only hidden_act='gelu' (erf) is on the reference path")
        self.fc1 = nn.Linear(config.hidden_size, config.intermediate_size)
        self.fc2 = nn.Linear(config.intermediate_size, config.hidden_size)

    def forward(self, x, colscale=None, residual=None):
        h = ops.linear(x, self.fc1.weight, bias=self.fc1.bias, act="gelu")
        return ops.linear(h, self.fc2.weight, bias=self.fc2.bias, colscale=colscale, residual=residual)


class InternVisionEncoderLayer(nn.Module):
    def __init__(self, config, drop_path_rate=0.0):
        super().__init__()
        self.embed_dim = config.hidden_size
        self.attn = InternAttention(config)
        self.mlp = InternMLP(config)
        self.norm1 = InternRMSNorm(self.embed_dim, eps=config.layer_norm_eps)
        self.norm2 = InternRMSNorm(self.embed_dim, eps=config.layer_norm_eps)
        self.ls1 = nn.Parameter(config.initializer_factor * torch.ones(self.embed_dim))
        self.ls2 = nn.Parameter(config.initializer_factor * torch.ones(self.embed_dim))

    def forward(self, x):
        x = self.attn(self.norm1(x), colscale=self.ls1, residual=x)
        return self.mlp(self.norm2(x), colscale=self.ls2, residual=x)


class InternVisionEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.layers = nn.ModuleList([InternVisionEncoderLayer(config) for _ in range(config.num_hidden_layers)])

    def forward(self, inputs_embeds, output_hidden_states=None):
        states = () if output_hidden_states else None
        x = inputs_embeds
        for layer in self.layers:
            if output_hidden_states:
                states = states + (x,)
            x = layer(x)
        if output_hidden_states:
            states = states + (x,)
        return SimpleNamespace(last_hidden_state=x, hidden_states=states)


class B200InternVisionModel(nn.Module):
    """Same call contract as the reference InternVisionModel.forward (:305-343)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = InternVisionEmbeddings(config)
        self.encoder = InternVisionEncoder(config)

    @property
    def dtype(self):
        return self.embeddings.position_embedding.dtype

    def get_input_embeddings(self):
        return self.embeddings

    @torch.no_grad()
    def forward(self, pixel_values=None, output_hidden_states=None, return_dict=None, pixel_embeds=None):
        if pixel_values is None and pixel_embeds is None:
            raise ValueError("You have to specify pixel_values or pixel_embeds")
        if pixel_embeds is not None:
            h = pixel_embeds
        elif pixel_values.dim() == 4:
            h = self.embeddings(pixel_values)
        else:
            raise ValueError(f"wrong pixel_values size: {pixel_values.shape}")
        if output_hidden_states is None:
            output_hidden_states = self.config.output_hidden_states
        enc = self.encoder(h, output_hidden_states=output_hidden_states)
        return SimpleNamespace(last_hidden_state=enc.last_hidden_state, pooler_output=enc.last_hidden_state[:, 0, :],
                               hidden_states=enc.hidden_states, attentions=None)
