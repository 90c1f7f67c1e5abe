"""UniPose's image backbone on the H100 kernels: the reference's own `SwinTransformer` + `Joiner`
(unipose/modeling_unipose.py:1212-1226 Joiner, :1277-1355 WindowAttention, :1357-1454 SwinTransformerBlock,
:1456-1494 PatchMerging, :1496-1595 BasicLayer, :1597-1636 PatchEmbed, :1638-1858 SwinTransformer, :4082-4120 / :4162-4222
builders), inference path.

Parameters live under the reference's names (`patch_embed.proj / .norm`, `layers.{i}.blocks.{j}.norm1 / .attn.qkv /
.attn.proj / .attn.relative_position_bias_table / .attn.relative_position_index / .norm2 / .mlp.fc1 / .mlp.fc2`,
`layers.{i}.downsample.reduction / .norm`, `norm{i}`), so `unipose.backbone.0.*` checkpoints load key for key.

The arithmetic is the Grounding-DINO Swin's (`swin.py`): per block ONE LayerNorm + pad + roll + window-partition gather,
packed q|k|v GEMM (+bias; already packed in the reference), window attention with the additive fp32 slab
(relative-position bias + the 0 / -100 shift mask of BasicLayer.forward), ONE gather back, proj GEMM with the shortcut
as fused residual, LayerNorm, fc1 GEMM + exact GELU, fc2 GEMM + residual; patch merging = 2x2 gather + LayerNorm(4C)
in one pass + reduction GEMM.  The reference scales q before q k^T; we scale the scores (same value up to rounding).

`build_backbone('internimage_h')` puts UniPose's copy of InternImage-H (:4675-4893, out indices (1, 2, 3)) behind the same
interface (`B200UniPoseInternImage`, the module tree of `internimage.B200InternImage`).

`B200Joiner(backbone)(tensors, mask)` returns what `Joiner.forward(NestedTensor)` returns: [(map NCHW, mask)] per
out index -- masks by nearest `F.interpolate` of the padding mask (:1847-1850) -- and the `PositionEmbeddingSineHW` of every
mask cast to the map dtype (:1223).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .internimage import INTERNIMAGE_H, B200InternImage
from .swin import _shift_mask, _window_reverse, _window_rows

SWIN_PRESETS = {                                                     # build_swin_transformer (:4082-4120)
    "swin_T_224_1k": dict(embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=7),
    "swin_B_224_22k": dict(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=7),
    "swin_B_384_22k": dict(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=12),
    "swin_L_224_22k": dict(embed_dim=192, depths=[2, 2, 18, 2], num_heads=[6, 12, 24, 48], window_size=7),
    "swin_L_384_22k": dict(embed_dim=192, depths=[2, 2, 18, 2], num_heads=[6, 12, 24, 48], window_size=12),
}


class _PatchEmbed(nn.Module):
    def __init__(self, patch_size, in_chans, embed_dim, patch_norm):
        super().__init__()
        self.patch_size = (patch_size, patch_size)
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = nn.LayerNorm(embed_dim) if patch_norm else None


class _WindowAttention(nn.Module):
    def __init__(self, dim, window_size, num_heads, qkv_bias):
        super().__init__()
        self.window_size, self.num_heads = (window_size, window_size), num_heads
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, num_heads))
        c = torch.stack(torch.meshgrid(torch.arange(window_size), torch.arange(window_size), indexing="ij")).flatten(1)
        rel = (c[:, :, None] - c[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += window_size - 1
        rel[:, :, 1] += window_size - 1
        rel[:, :, 0] *= 2 * window_size - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(dim, hidden), nn.Linear(hidden, dim)


class _Block(nn.Module):
    def __init__(self, dim, num_heads, window_size, shift_size, mlp_ratio, qkv_bias):
        super().__init__()
        self.window_size, self.shift_size, self.num_heads = window_size, shift_size, num_heads
        self.norm1 = nn.LayerNorm(dim)
        self.attn = _WindowAttention(dim, window_size, num_heads, qkv_bias)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio))


class _PatchMerging(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(4 * dim)


class _BasicLayer(nn.Module):
    def __init__(self, dim, depth, num_heads, window_size, mlp_ratio, qkv_bias, downsample):
        super().__init__()
        self.blocks = nn.ModuleList([_Block(dim, num_heads, window_size, 0 if i % 2 == 0 else window_size // 2, mlp_ratio,
                                            qkv_bias) for i in range(depth)])
        self.downsample = _PatchMerging(dim) if downsample else None


class B200UniPoseSwin(nn.Module):
    """`SwinTransformer(pretrain_img_size, patch_size=4, ..., out_indices, dilation=False)` of the reference, inference."""

    def __init__(self, pretrain_img_size=224, patch_size=4, in_chans=3, embed_dim=96, depths=(2, 2, 6, 2),
                 num_heads=(3, 6, 12, 24), window_size=7, mlp_ratio=4., qkv_bias=True, qk_scale=None, ape=False,
                 patch_norm=True, out_indices=(0, 1, 2, 3), dilation=False, **unused):
        super().__init__()
        if ape:
            raise NotImplementedError("absolute position embedding (ape=True; no reference preset uses it)")
        if dilation:
            raise NotImplementedError("dilation=True (build_backbone passes dilation=False, :4199)")
        if qk_scale is not None:
            raise NotImplementedError("qk_scale override")
        self.num_layers, self.embed_dim, self.out_indices = len(depths), embed_dim, tuple(out_indices)
        self.patch_embed = _PatchEmbed(patch_size, in_chans, embed_dim, patch_norm)
        self.num_features = [int(embed_dim * 2 ** i) for i in range(self.num_layers)]
        self.layers = nn.ModuleList([
            _BasicLayer(self.num_features[i], depths[i], num_heads[i], window_size, mlp_ratio, qkv_bias,
                        downsample=i < self.num_layers - 1) for i in range(self.num_layers)])
        for i in self.out_indices:
            self.add_module(f"norm{i}", nn.LayerNorm(self.num_features[i]))
        self._idx, self._bias = {}, {}

    # ---- cached integer plumbing / bias slabs ----
    def _rows(self, H, W, ws, shift, device):
        key = (H, W, ws, shift, str(device))
        if key not in self._idx:
            fwd, inv, Hp, Wp = _window_rows(H, W, ws, shift, device)
            mask = _shift_mask(Hp, Wp, ws, shift, device) if shift > 0 else None            # BasicLayer.forward (:1563-1580)
            self._idx[key] = (fwd, inv, Hp, Wp, mask)
        return self._idx[key]

    def _attn_bias(self, blk, mask, tag):
        at = blk.attn
        t = at.relative_position_bias_table
        key = (id(blk), tag, t.data_ptr(), str(t.device), t._version)
        if key not in self._bias:
            T = blk.window_size * blk.window_size
            rel = t[at.relative_position_index.view(-1)].view(T, T, -1).permute(2, 0, 1).float()   # [heads, T, T]
            self._bias[key] = (rel[None] if mask is None else rel[None] + mask[:, None]).contiguous()
        return self._bias[key]

    # ---- forward pieces ----
    @torch.no_grad()
    def _embed(self, x):
        pe = self.patch_embed
        ph, pw = pe.patch_size
        if x.shape[3] % pw:                                                                  # PatchEmbed.forward (:1623-1626)
            x = F.pad(x, (0, pw - x.shape[3] % pw))
        if x.shape[2] % ph:
            x = F.pad(x, (0, 0, 0, ph - x.shape[2] % ph))
        B, Cin, Hh, W = x.shape
        h, w = Hh // ph, W // pw
        rows = x.view(B, Cin, h, ph, w, pw).permute(0, 2, 4, 1, 3, 5).reshape(B, h * w, Cin * ph * pw)
        wgt = pe.proj.weight.view(pe.proj.out_channels, -1)
        if rows.shape[-1] % 8:                                                               # GEMM rows: 16-byte multiples
            padk = 8 - rows.shape[-1] % 8
            rows, wgt = F.pad(rows, (0, padk)), F.pad(wgt, (0, padk))
        y = ops.linear(rows.contiguous(), wgt.contiguous(), bias=pe.proj.bias)
        if pe.norm is not None:
            y = ops.layernorm(y, pe.norm.weight, pe.norm.bias, pe.norm.eps)
        return y, (h, w)

    @torch.no_grad()
    def _block(self, blk, x, H, W):
        B, N, C = x.shape
        ws, shift, nH = blk.window_size, blk.shift_size, blk.num_heads
        D = C // nH
        fwd, inv, Hp, Wp, mask = self._rows(H, W, ws, int(shift), x.device)
        bias = self._attn_bias(blk, mask, (H, W))
        n1 = blk.norm1
        win = ops.layernorm_gather(x.contiguous(), fwd, n1.weight, n1.bias, n1.eps)          # [B, nW*T, C], window-major
        T, nW = ws * ws, (Hp // ws) * (Wp // ws)
        qkv = ops.linear(win, blk.attn.qkv.weight, bias=blk.attn.qkv.bias).view(B * nW, T, 3, nH, D)
        ctx = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], scale=1.0 / math.sqrt(D), attn_bias=bias)
        ctx = _window_reverse(self._idx, ctx.view(B * nW * T, C), inv, B, nW * T, N)
        x = ops.linear(ctx, blk.attn.proj.weight, bias=blk.attn.proj.bias, residual=x)
        n2 = blk.norm2
        h = ops.layernorm(x, n2.weight, n2.bias, n2.eps)
        h = ops.linear(h, blk.mlp.fc1.weight, bias=blk.mlp.fc1.bias, act="gelu")
        return ops.linear(h, blk.mlp.fc2.weight, bias=blk.mlp.fc2.bias, residual=x)

    @torch.no_grad()
    def _merge(self, ds, x, H, W):
        B, N, C = x.shape
        if (x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous() and H % 2 == 0 and W % 2 == 0
                and ds.norm.weight.dtype == torch.bfloat16 and C % 8 == 0 and 4 * C <= 16384):
            y = ops.pixel_shuffle_rows(x, 0, ds.norm.weight, ds.norm.bias, ds.norm.eps, grid=(H, W), order=1)
            return ops.linear(y, ds.reduction.weight)
        x = x.view(B, H, W, C)
        if H % 2 or W % 2:
            x = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
        x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)   # PatchMerging (:1484-1488)
        x = x.reshape(B, -1, 4 * C)
        x = ops.layernorm(x, ds.norm.weight, ds.norm.bias, ds.norm.eps)
        return ops.linear(x, ds.reduction.weight)

    @torch.no_grad()
    def forward_raw(self, x):
        """:1779-1808 -- the tuple of NCHW maps (views of channels-last storage) of the out indices."""
        x, (H, W) = self._embed(x)
        outs = []
        for i, layer in enumerate(self.layers):
            for blk in layer.blocks:
                x = self._block(blk, x, H, W)
            if i in self.out_indices:
                n = getattr(self, f"norm{i}")
                outs.append(ops.layernorm(x, n.weight, n.bias, n.eps).view(x.shape[0], H, W, -1).permute(0, 3, 1, 2))
            if layer.downsample is not None:
                x = self._merge(layer.downsample, x, H, W)
                H, W = (H + 1) // 2, (W + 1) // 2
        return tuple(outs)

    @torch.no_grad()
    def forward(self, tensors, mask):
        """:1811-1852 with the NestedTensor unpacked: {idx: (map NCHW, mask [bs, h, w] bool, True = padding)}."""
        outs = self.forward_raw(tensors)
        return {i: (o, F.interpolate(mask[None].float(), size=o.shape[-2:]).to(torch.bool)[0]) for i, o in enumerate(outs)}


class B200Joiner(nn.Sequential):
    """`Joiner(backbone, position_embedding)` (:1212-1226): index 0 / 1 like the reference (its state-dict prefix `0.`)."""

    def __init__(self, backbone, position_embedding):
        super().__init__(backbone, position_embedding)
        self.num_channels = None

    @torch.no_grad()
    def forward(self, tensors, mask):
        xs = self[0](tensors, mask)
        out, pos = [], []
        for _, (t, m) in xs.items():
            out.append((t, m))
            pos.append(self[1](m).to(t.dtype))
        return out, pos


class B200UniPoseInternImage(B200InternImage):
    """UniPose's own copy of InternImage (modeling_unipose.py:4675-4864: the class of gd.py whose `forward(NestedTensor)` returns
    {idx: NestedTensor(map NCHW, interpolated padding mask)}).  Same module tree as `internimage.B200InternImage`, so the
    state-dict keys under the Joiner are the reference's (`0.patch_embed.*`, `0.levels.*`)."""

    @torch.no_grad()
    def forward(self, tensors, mask):
        outs = B200InternImage.forward(self, tensors)                                       # channels-last [B, h, w, C] maps
        res = {}
        for i, o in enumerate(outs):
            o = o.permute(0, 3, 1, 2)                                                        # NCHW view of the channels-last storage
            res[i] = (o, F.interpolate(mask[None].float(), size=o.shape[-2:]).to(torch.bool)[0])
        return res


def build_internimage_h(**overrides):
    """modeling_unipose.py:4866-4893: the InternImage-H preset with out_indices (1, 2, 3); `num_features` pinned to the H widths."""
    cfg = dict(INTERNIMAGE_H)
    cfg.update(out_indices=(1, 2, 3), channels_last_out=True)
    cfg.update(overrides)
    m = B200UniPoseInternImage(**cfg)
    if not overrides:
        m.num_features = [320, 640, 1280, 2560]
    return m


def build_backbone(backbone="swin_T_224_1k", return_interm_indices=(1, 2, 3), hidden_dim=256, pe_temperatureH=20,
                   pe_temperatureW=20, **swin_overrides):
    """`build_backbone(args)` (:4162-4222) for the Swin presets and 'internimage_h' + `build_position_encoding` ('sine',
    :4224-4233).  Keyword overrides (tests) replace preset fields of the chosen backbone."""
    from .unipose import PositionEmbeddingSineHW
    if list(return_interm_indices) not in ([0, 1, 2, 3], [1, 2, 3], [3]):
        raise ValueError("return_interm_indices must be [0, 1, 2, 3], [1, 2, 3] or [3]")
    if backbone == "internimage_h":                                                        # :4203-4205
        body = build_internimage_h(**swin_overrides)
        joiner = B200Joiner(body, PositionEmbeddingSineHW(hidden_dim // 2, pe_temperatureH, pe_temperatureW, normalize=True))
        joiner.num_channels = list(body.num_features[4 - len(return_interm_indices):])
        if len(joiner.num_channels) != len(body.out_indices):                              # the reference's assert (:4209-4211)
            raise ValueError(f"internimage_h returns levels {body.out_indices}: return_interm_indices must have as many entries")
        return joiner
    if backbone not in SWIN_PRESETS:
        raise NotImplementedError(f"backbone {backbone!r}: the Swin presets and 'internimage_h' are built here (the ResNet "
                                  "backbones of :4187-4195 are torchvision models outside this path)")
    kw = dict(SWIN_PRESETS[backbone])
    kw.update(swin_overrides)
    swin = B200UniPoseSwin(pretrain_img_size=int(backbone.split("_")[-2]), out_indices=tuple(return_interm_indices),
                           dilation=False, **kw)
    joiner = B200Joiner(swin, PositionEmbeddingSineHW(hidden_dim // 2, pe_temperatureH, pe_temperatureW, normalize=True))
    joiner.num_channels = swin.num_features[4 - len(return_interm_indices):]
    return joiner
