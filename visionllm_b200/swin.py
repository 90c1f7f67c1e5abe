"""Swin Transformer backbone of the Grounding-DINO stage (SURVEY 8a row a13) on the H100 kernels.

The reference builds it with HF `AutoBackbone.from_config(config.backbone_config)`
(grounding_dino/modeling_ov_grounding_dino_mask_dn.py:471-504) -- third-party `transformers.models.swin.modeling_swin`
(SwinBackbone / SwinEncoder / SwinStage / SwinLayer / SwinSelfAttention / SwinPatchMerging), whose arithmetic this
module restates.  Parameters live in the HF sub-modules themselves (`embeddings`, `encoder`, `hidden_states_norms`),
so the state dict is the HF one key for key and `model.backbone.conv_encoder.model.*` checkpoints load unchanged.

Dataflow per SwinLayer, all row-major [tokens, C] bf16:
  LayerNorm kernel -> ONE gather (pad-to-window + cyclic shift + window partition folded into an int64 row index)
  -> packed q|k|v GEMM (+bias) -> fused window attention (D=32, 49 or 144 tokens, additive fp32 bias slab
  [windows, heads, T, T] = relative-position bias + shifted-window mask, read in place through `attn_bias`)
  -> ONE gather back (window reverse + un-shift + crop) -> out-proj GEMM with the shortcut as fused residual
  -> LayerNorm -> fc1 GEMM + exact GELU epilogue -> fc2 GEMM with fused residual.
Padded tokens are zero rows that DO take part in attention as keys, exactly as in HF (only the shift mask is applied).
The int64 index tensors and bias slabs are cached per (H, W, window, shift) / per layer.

Feature maps are returned channels-last ([B, H, W, C], tagged `_b200_nhwc`) for our neck; `nchw=True` gives HF's layout.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops


def _window_rows(H, W, ws, shift, device):
    """Row indices implementing pad -> roll(-shift) -> window_partition and its inverse.
    fwd [nW*ws*ws]: source row in the H*W token list for every window slot (H*W = the appended zero row);
    inv [H*W]: window slot holding each token after window_reverse -> roll(+shift) -> crop."""
    Hp, Wp = (H + ws - 1) // ws * ws, (W + ws - 1) // ws * ws
    ys = torch.arange(Hp, device=device)
    xs = torch.arange(Wp, device=device)
    sy, sx = (ys + shift) % Hp, (xs + shift) % Wp                        # rolled[y] = padded[(y + shift) % Hp]
    src = sy[:, None] * W + sx[None, :]
    src = torch.where((sy[:, None] < H) & (sx[None, :] < W), src, torch.full_like(src, H * W))
    fwd = src.view(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1)
    slot = torch.arange(Hp * Wp, device=device).view(Hp // ws, Wp // ws, ws, ws).permute(0, 2, 1, 3).reshape(Hp, Wp)
    # un-shift: out[y] = shifted[(y - shift) % Hp]
    uy, ux = (ys - shift) % Hp, (xs - shift) % Wp
    inv = slot[uy][:, ux][:H, :W].reshape(-1)
    return fwd, inv, Hp, Wp


def _shift_mask(Hp, Wp, ws, shift, device):
    """SwinLayer.get_attn_mask: 0 / -100 per window pair pattern, [nW, T, T] fp32."""
    img = torch.zeros((Hp, Wp), dtype=torch.float32, device=device)
    cnt = 0
    for hs in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
        for wsl in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
            img[hs, wsl] = cnt
            cnt += 1
    mw = img.view(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def _window_reverse(cache, ctx2d, inv, B, slots, N):
    """window_reverse + un-shift + crop as ONE row gather ctx2d[b * slots + inv[n]] -> [B, N, C] (`vllm_gather_rows_bf16`,
    flat 16-byte-vector kernel for these narrow rows); the batched int64 index is cached per (geometry, batch)."""
    key = ("flat", inv.data_ptr(), B, slots)
    if key not in cache:
        cache[key] = (torch.arange(B, device=inv.device)[:, None] * slots + inv[None, :]).reshape(-1).contiguous()
    return ops.gather_rows(ctx2d, cache[key]).view(B, N, ctx2d.shape[-1])


class B200SwinBackbone(nn.Module):
    def __init__(self, config):
        super().__init__()
        from transformers.models.swin.modeling_swin import SwinBackbone
        hf = SwinBackbone(config)
        self.config = config
        self.embeddings, self.encoder, self.hidden_states_norms = hf.embeddings, hf.encoder, hf.hidden_states_norms
        self.stage_names, self.out_features, self.channels = hf.stage_names, hf.out_features, hf.channels
        if config.hidden_act != "gelu":
            raise NotImplementedError("Swin MLP activation other than exact GELU")
        if self.embeddings.position_embeddings is not None:
            raise NotImplementedError("absolute position embeddings")
        self._idx, self._packed = {}, {}

    # ---- cached integer / weight plumbing ----
    def _rows(self, H, W, ws, shift, device):
        key = (H, W, ws, shift, str(device))
        if key not in self._idx:
            fwd, inv, Hp, Wp = _window_rows(H, W, ws, shift, device)
            mask = _shift_mask(Hp, Wp, ws, shift, device) if shift > 0 else None
            self._idx[key] = (fwd, inv, Hp, Wp, mask)
        return self._idx[key]

    def _layer_pack(self, layer, mask, tag):
        """(packed qkv weight [3C, C], bias [3C], attn_bias [nW or 1, heads, T, T] fp32)."""
        sa = layer.attention.self
        key = (id(layer), tag, sa.query.weight.data_ptr(), sa.query.weight.dtype, str(sa.query.weight.device),
               sa.query.weight._version, sa.relative_position_bias_table._version)
        if key not in self._packed:
            w = torch.cat((sa.query.weight, sa.key.weight, sa.value.weight), 0).contiguous()
            b = None if sa.query.bias is None else torch.cat((sa.query.bias, sa.key.bias, sa.value.bias), 0).contiguous()
            T = sa.window_size[0] * sa.window_size[1]
            rel = sa.relative_position_bias_table[sa.relative_position_index.view(-1)].view(T, T, -1)
            rel = rel.permute(2, 0, 1).float()                                           # [heads, T, T]
            bias = rel[None] if mask is None else rel[None] + mask[:, None]
            self._packed[key] = (w, b, bias.contiguous())
        return self._packed[key]

    # ---- forward pieces ----
    @torch.no_grad()
    def _embed(self, pixel_values):
        pe = self.embeddings.patch_embeddings
        ph, pw = pe.patch_size
        x = pe.maybe_pad(pixel_values, pixel_values.shape[2], pixel_values.shape[3])
        B, Cin, Hh, W = x.shape
        h, w = Hh // ph, W // pw
        rows = x.view(B, Cin, h, ph, w, pw).permute(0, 2, 4, 1, 3, 5).reshape(B, h * w, Cin * ph * pw)   # (c, ky, kx) = conv weight order
        conv = pe.projection
        wgt = conv.weight.view(conv.out_channels, -1)
        if rows.shape[-1] % 8:                                             # GEMM rows must be 16-byte multiples
            padk = 8 - rows.shape[-1] % 8
            rows, wgt = nn.functional.pad(rows, (0, padk)), nn.functional.pad(wgt, (0, padk))
        y = ops.linear(rows.contiguous(), wgt.contiguous(), bias=conv.bias)
        n = self.embeddings.norm
        return ops.layernorm(y, n.weight, n.bias, n.eps), (h, w)

    @torch.no_grad()
    def _layer(self, layer, x, H, W):
        B, N, C = x.shape
        ws, shift = layer.window_size, layer.shift_size                  # always_partition=True: never shrunk
        sa = layer.attention.self
        nH, D = sa.num_attention_heads, sa.attention_head_size
        fwd, inv, Hp, Wp, mask = self._rows(H, W, ws, int(shift), x.device)
        w_qkv, b_qkv, bias = self._layer_pack(layer, mask, (H, W))
        ln = layer.layernorm_before
        # layernorm_before + zero pad + roll + window partition in ONE pass: fwd[j] = raster row of window slot j (N = pad)
        win = ops.layernorm_gather(x.contiguous(), fwd, ln.weight, ln.bias, ln.eps)     # [B, nW*T, C], window-major
        T = ws * ws
        nW = (Hp // ws) * (Wp // ws)
        qkv = ops.linear(win, w_qkv, bias=b_qkv).view(B * nW, T, 3, nH, D)
        ctx = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], scale=1.0 / math.sqrt(D), attn_bias=bias)
        ctx = _window_reverse(self._idx, ctx.view(B * nW * T, C), inv, B, nW * T, N)   # back to raster order, pads dropped
        dense = layer.attention.output.dense
        x = ops.linear(ctx, dense.weight, bias=dense.bias, residual=x)
        ln2 = layer.layernorm_after
        h = ops.layernorm(x, ln2.weight, ln2.bias, ln2.eps)
        fc1, fc2 = layer.intermediate.dense, layer.output.dense
        h = ops.linear(h, fc1.weight, bias=fc1.bias, act="gelu")
        return ops.linear(h, fc2.weight, bias=fc2.bias, residual=x)

    @torch.no_grad()
    def _merge(self, ds, x, H, W):
        B, N, C = x.shape
        if (x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous() and H % 2 == 0 and W % 2 == 0
                and ds.norm.weight.dtype == torch.bfloat16 and C % 8 == 0 and 4 * C <= 16384):
            # the 2x2 gather (HF SwinPatchMerging's cat order) and the LayerNorm(4C) in ONE pass (csrc/seqglue.cu)
            y = ops.pixel_shuffle_rows(x, 0, ds.norm.weight, ds.norm.bias, ds.norm.eps, grid=(H, W), order=1)
            return ops.linear(y, ds.reduction.weight)
        x = x.view(B, H, W, C)
        if H % 2 or W % 2:
            x = nn.functional.pad(x, (0, 0, 0, W % 2, 0, H % 2))
        x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
        x = x.reshape(B, -1, 4 * C)
        x = ops.layernorm(x, ds.norm.weight, ds.norm.bias, ds.norm.eps)
        return ops.linear(x, ds.reduction.weight)

    @torch.no_grad()
    def forward(self, pixel_values, nchw=False, **unused):
        x, (H, W) = self._embed(pixel_values)
        maps = []
        for i, stage in enumerate(self.encoder.layers):
            for blk in stage.blocks:
                x = self._layer(blk, x, H, W)
            name = self.stage_names[i + 1]
            if name in self.out_features:
                n = self.hidden_states_norms[name]
                f = ops.layernorm(x, n.weight, n.bias, n.eps).view(x.shape[0], H, W, -1)
                if nchw:
                    f = f.permute(0, 3, 1, 2).contiguous()
                else:
                    f._b200_nhwc = True
                maps.append(f)
            if stage.downsample is not None:
                x = self._merge(stage.downsample, x, H, W)
                H, W = (H + 1) // 2, (W + 1) // 2
        return SimpleNamespace(feature_maps=tuple(maps))
