"""H100-native InternImage backbone (SURVEY.md 8a-a13, second option: InternImage-H for the Grounding-DINO stage).

Drop-in for the reference classes `InternImage` / `build_internimage_h` / `GroundingDinoInternImageBackbone`
(visionllmv2/model/grounding_dino/modeling_ov_grounding_dino_mask_dn.py:4689-5209) and the `DCNv3` module they are
built from (visionllmv2/model/ops_dcnv3/modules/dcnv3.py:211-351): the same state-dict keys (the reference wraps every
norm in an `nn.Sequential` of layout permutes, so the LayerNorms live under `...norm1.0`, `...dw_conv.1.1`,
`patch_embed.norm1.1`, ...; the containers are rebuilt here key for key), the same constructor arguments, the same
forward contract (`forward(x[B,3,H,W]) -> [level maps]`).

Execution on our kernels, channels-last throughout (the reference permutes to NCHW and back around every conv):
  stem / downsample 3x3-s2 convs   tap-gather + wgmma GEMM (+bias)                     ops.linear
  LayerNorms                       row kernel; the `LN -> GELU` tail of the depthwise branch in ONE pass
  depthwise 5x5 (3x3) conv         csrc/dwconv.cu (register-tiled, NHWC)                  ops.dwconv_nhwc
  input_proj                       GEMM -> fp32 (the core op is fp32, dcnv3.py:331-340)
  offset | mask | centre-scale     ONE packed GEMM -> fp32 (the reference issues three)
  DCNv3 core                       csrc/dcnv3.cu through visionllm_b200.dcnv3.dcnv3_forward
  output_proj, MLP fc1(+GELU)/fc2  GEMM epilogues
  slices / 9-way mask softmax / sigmoid            ONE pass over the packed projection  ops.dcnv3_prep
  centre-feature blend + bf16 cast                 ONE pass                              ops.dcnv3_blend
  post-norm residual  x + LN(.)                    inside the LayerNorm pass
Forward only (the GDINO stage of the eval path); DropPath / dropout are identities at eval like in the reference.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import dcnv3 as dcn_ext
from . import ops


class _Permute(nn.Identity):
    """Parameter-free placeholder for the reference's to_channels_first / to_channels_last (keeps Sequential indices)."""


def build_norm_layer(dim, norm_layer, in_format="channels_last", out_format="channels_last", eps=1e-6):
    """Same container layout as the reference helper (gd.py:4654-4675): the LayerNorm's index inside the Sequential
    depends on the formats, and that index is part of the checkpoint key."""
    if norm_layer != "LN":
        raise NotImplementedError(f"build_norm_layer does not support {norm_layer} (InternImage-H uses LN)")
    layers = []
    if in_format == "channels_first":
        layers.append(_Permute())
    layers.append(nn.LayerNorm(dim, eps=eps))
    if out_format == "channels_first":
        layers.append(_Permute())
    return nn.Sequential(*layers)


def _ln(seq):
    for m in seq:
        if isinstance(m, nn.LayerNorm):
            return m
    raise RuntimeError("no LayerNorm in container")


def _apply_ln(seq, x, gelu=False, residual=None):
    ln = _ln(seq)
    return ops.layernorm(x, ln.weight, ln.bias, ln.eps, gelu=gelu, residual=residual)


class _Cache:
    """Derived operands (repacked conv weights, packed projections) rebuilt only when a source tensor changes."""

    def __init__(self):
        self.key, self.val = None, None

    def get(self, tensors, dtype, build):
        key = tuple((t.data_ptr(), t._version) for t in tensors if t is not None) + (dtype,)
        if self.key != key:
            self.key, self.val = key, build()
        return self.val


def conv_s2_rows(x, conv, cache):
    """3x3 stride-2 padding-1 Conv2d over a channels-last map as a tap gather + ONE GEMM.  Input channels are padded
    to a multiple of 8 (the RGB stem) so GEMM rows keep a 16-byte pitch."""
    B, Hh, W, C = x.shape
    k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    Cp = (C + 7) // 8 * 8

    def build():
        w = conv.weight.detach().permute(0, 2, 3, 1)                       # [Cout, k, k, Cin]
        if Cp != C:
            w = F.pad(w, (0, Cp - C))
        return w.reshape(conv.out_channels, k * k * Cp).to(x.dtype).contiguous()
    w_rows = cache.get((conv.weight,), x.dtype, build)
    Ho, Wo = (Hh + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    xp = F.pad(x, (0, Cp - C, p, p, p, p))
    taps = [xp[:, dy:dy + s * (Ho - 1) + 1:s, dx:dx + s * (Wo - 1) + 1:s, :] for dy in range(k) for dx in range(k)]
    rows = torch.cat(taps, -1).reshape(B * Ho * Wo, k * k * Cp)
    bias = conv.bias.detach().to(x.dtype) if conv.bias is not None else None
    return ops.linear(rows, w_rows, bias=bias).view(B, Ho, Wo, conv.out_channels)


class StemLayer(nn.Module):
    """gd.py:4689-4726: conv3x3 s2 -> LN -> GELU -> conv3x3 s2 -> LN, output channels-last."""

    def __init__(self, in_chans=3, out_chans=96, act_layer="GELU", norm_layer="LN"):
        super().__init__()
        if act_layer != "GELU":
            raise NotImplementedError("StemLayer: GELU only")
        self.conv1 = nn.Conv2d(in_chans, out_chans // 2, kernel_size=3, stride=2, padding=1)
        self.norm1 = build_norm_layer(out_chans // 2, norm_layer, "channels_first", "channels_first")
        self.act = nn.GELU()
        self.conv2 = nn.Conv2d(out_chans // 2, out_chans, kernel_size=3, stride=2, padding=1)
        self.norm2 = build_norm_layer(out_chans, norm_layer, "channels_first", "channels_last")
        self._c1, self._c2 = _Cache(), _Cache()

    def forward(self, x):                                                   # x: [B, 3, H, W]
        x = x.permute(0, 2, 3, 1).contiguous()
        x = conv_s2_rows(x, self.conv1, self._c1)
        x = _apply_ln(self.norm1, x, gelu=True)
        x = conv_s2_rows(x, self.conv2, self._c2)
        return _apply_ln(self.norm2, x)


class DownsampleLayer(nn.Module):
    """gd.py:4729-4750: conv3x3 s2 (C -> 2C, no bias) -> LN."""

    def __init__(self, channels, norm_layer="LN"):
        super().__init__()
        self.conv = nn.Conv2d(channels, 2 * channels, kernel_size=3, stride=2, padding=1, bias=False)
        self.norm = build_norm_layer(2 * channels, norm_layer, "channels_first", "channels_last")
        self._c = _Cache()

    def forward(self, x):
        return _apply_ln(self.norm, conv_s2_rows(x, self.conv, self._c))


class MLPLayer(nn.Module):
    """gd.py:4753-4783."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer="GELU", drop=0.):
        super().__init__()
        if act_layer != "GELU":
            raise NotImplementedError("MLPLayer: GELU only")
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)

    def forward(self, x):
        return ops.linear(ops.linear(x, self.fc1.weight, bias=self.fc1.bias, act="gelu"), self.fc2.weight,
                          bias=self.fc2.bias)


class DCNv3(nn.Module):
    """The DCNv3 module (ops_dcnv3/modules/dcnv3.py:211-351), parameters named like the reference's."""

    def __init__(self, channels=64, kernel_size=3, dw_kernel_size=None, stride=1, pad=1, dilation=1, group=4,
                 offset_scale=1.0, act_layer="GELU", norm_layer="LN", center_feature_scale=False):
        super().__init__()
        if channels % group != 0:
            raise ValueError(f"channels must be divisible by group, but got {channels} and {group}")
        if act_layer != "GELU":
            raise NotImplementedError("DCNv3: GELU only")
        dw_kernel_size = dw_kernel_size if dw_kernel_size is not None else kernel_size
        self.offset_scale, self.channels, self.kernel_size, self.dw_kernel_size = offset_scale, channels, kernel_size, dw_kernel_size
        self.stride, self.dilation, self.pad, self.group = stride, dilation, pad, group
        self.group_channels = channels // group
        self.center_feature_scale = center_feature_scale
        self.dw_conv = nn.Sequential(
            nn.Conv2d(channels, channels, kernel_size=dw_kernel_size, stride=1, padding=(dw_kernel_size - 1) // 2,
                      groups=channels),
            build_norm_layer(channels, norm_layer, "channels_first", "channels_last"),
            nn.GELU())
        self.offset = nn.Linear(channels, group * kernel_size * kernel_size * 2)
        self.mask = nn.Linear(channels, group * kernel_size * kernel_size)
        self.input_proj = nn.Linear(channels, channels)
        self.output_proj = nn.Linear(channels, channels)
        self._reset_parameters()
        if center_feature_scale:
            self.center_feature_scale_proj_weight = nn.Parameter(torch.zeros((group, channels), dtype=torch.float))
            self.center_feature_scale_proj_bias = nn.Parameter(torch.zeros(group, dtype=torch.float))
        self._dw, self._packed = _Cache(), _Cache()

    def _reset_parameters(self):
        for lin in (self.offset, self.mask):
            nn.init.constant_(lin.weight.data, 0.)
            nn.init.constant_(lin.bias.data, 0.)
        for lin in (self.input_proj, self.output_proj):
            nn.init.xavier_uniform_(lin.weight.data)
            nn.init.constant_(lin.bias.data, 0.)

    def _query_proj(self, dtype):
        """offset | mask | centre-feature-scale projections as ONE [G*K*3 (+G), C] operand."""
        ws = [self.offset.weight, self.mask.weight, self.offset.bias, self.mask.bias]
        if self.center_feature_scale:
            ws += [self.center_feature_scale_proj_weight, self.center_feature_scale_proj_bias]

        def build():
            w = [self.offset.weight, self.mask.weight]
            b = [self.offset.bias, self.mask.bias]
            if self.center_feature_scale:
                w.append(self.center_feature_scale_proj_weight)
                b.append(self.center_feature_scale_proj_bias)
            wc = torch.cat([t.detach().to(dtype) for t in w], 0)
            bc = torch.cat([t.detach().to(dtype) for t in b], 0)
            pad = (-wc.shape[0]) % 4                      # fp32 GEMM output rows need a 16-byte pitch
            if pad:
                wc, bc = F.pad(wc, (0, 0, 0, pad)), F.pad(bc, (0, pad))
            return wc.contiguous(), bc.contiguous()
        return self._packed.get(ws, dtype, build)

    def forward(self, input):                                               # [N, H, W, C] channels-last
        N, Hh, W, C = input.shape
        G, K = self.group, self.kernel_size * self.kernel_size
        conv = self.dw_conv[0]
        k = self.dw_kernel_size
        wt = self._dw.get((conv.weight,), input.dtype,
                          lambda: conv.weight.detach().reshape(C, k * k).t().to(input.dtype).contiguous())
        x32 = ops.linear(input, self.input_proj.weight, bias=self.input_proj.bias, out_dtype=torch.float32)
        x1 = ops.dwconv_nhwc(input.contiguous(), wt, conv.bias.detach().to(input.dtype), k)
        x1 = _apply_ln(self.dw_conv[1], x1, gelu=True)
        wq, bq = self._query_proj(input.dtype)
        om = ops.linear(x1, wq, bias=bq, out_dtype=torch.float32)          # [N, H, W, G*K*2 | G*K | G]
        offset, mask, cfs = ops.dcnv3_prep(om, G, K, self.center_feature_scale)   # slices, 9-way softmax, sigmoid
        x = dcn_ext.dcnv3_forward(x32.view(N, Hh, W, C), offset, mask, self.kernel_size, self.kernel_size, self.stride,
                                  self.stride, self.pad, self.pad, self.dilation, self.dilation, G, self.group_channels,
                                  self.offset_scale, 256)
        x = ops.dcnv3_blend(x, x32.view(N, Hh, W, C), cfs, self.group_channels)    # centre-feature blend + bf16 cast
        return ops.linear(x, self.output_proj.weight, bias=self.output_proj.bias)


class InternImageLayer(nn.Module):
    """gd.py:4786-4883 (all four residual arrangements: plain / post_norm / res_post_norm, with or without gammas)."""

    def __init__(self, core_op, channels, groups, mlp_ratio=4., drop=0., drop_path=0., act_layer="GELU",
                 norm_layer="LN", post_norm=False, layer_scale=None, offset_scale=1.0, with_cp=False,
                 dw_kernel_size=None, res_post_norm=False, center_feature_scale=False):
        super().__init__()
        self.channels, self.groups, self.mlp_ratio = channels, groups, mlp_ratio
        self.norm1 = build_norm_layer(channels, "LN")
        self.post_norm = post_norm
        self.dcn = core_op(channels=channels, kernel_size=3, stride=1, pad=1, dilation=1, group=groups,
                           offset_scale=offset_scale, act_layer=act_layer, norm_layer=norm_layer,
                           dw_kernel_size=dw_kernel_size, center_feature_scale=center_feature_scale)
        self.norm2 = build_norm_layer(channels, "LN")
        self.mlp = MLPLayer(in_features=channels, hidden_features=int(channels * mlp_ratio), act_layer=act_layer, drop=drop)
        self.layer_scale = layer_scale is not None
        if self.layer_scale:
            self.gamma1 = nn.Parameter(layer_scale * torch.ones(channels))
            self.gamma2 = nn.Parameter(layer_scale * torch.ones(channels))
        self.res_post_norm = res_post_norm
        if res_post_norm:
            self.res_post_norm1 = build_norm_layer(channels, "LN")
            self.res_post_norm2 = build_norm_layer(channels, "LN")

    def forward(self, x):
        n1 = lambda t: _apply_ln(self.norm1, t)          # noqa: E731
        n2 = lambda t: _apply_ln(self.norm2, t)          # noqa: E731
        if not self.layer_scale:
            if self.post_norm:
                x = x + n1(self.dcn(x))
                return x + n2(self.mlp(x))
            if self.res_post_norm:
                x = _apply_ln(self.res_post_norm1, self.dcn(n1(x)), residual=x)
                return _apply_ln(self.res_post_norm2, self.mlp(n2(x)), residual=x)
            x = x + self.dcn(n1(x))
            return x + self.mlp(n2(x))
        g1, g2 = self.gamma1.to(x.dtype), self.gamma2.to(x.dtype)
        if self.post_norm:
            x = x + g1 * n1(self.dcn(x))
            return x + g2 * n2(self.mlp(x))
        x = x + g1 * self.dcn(n1(x))
        return x + g2 * self.mlp(n2(x))


class InternImageBlock(nn.Module):
    """gd.py:4886-4975."""

    def __init__(self, core_op, channels, depth, groups, downsample=True, mlp_ratio=4., drop=0., drop_path=0.,
                 act_layer="GELU", norm_layer="LN", post_norm=False, offset_scale=1.0, layer_scale=None,
                 with_cp=False, dw_kernel_size=None, post_norm_block_ids=None, res_post_norm=False,
                 center_feature_scale=False):
        super().__init__()
        self.channels, self.depth, self.post_norm, self.center_feature_scale = channels, depth, post_norm, center_feature_scale
        self.blocks = nn.ModuleList([
            InternImageLayer(core_op=core_op, channels=channels, groups=groups, mlp_ratio=mlp_ratio, drop=drop,
                             act_layer=act_layer, norm_layer=norm_layer, post_norm=post_norm, layer_scale=layer_scale,
                             offset_scale=offset_scale, dw_kernel_size=dw_kernel_size, res_post_norm=res_post_norm,
                             center_feature_scale=center_feature_scale) for _ in range(depth)])
        if not self.post_norm or center_feature_scale:
            self.norm = build_norm_layer(channels, "LN")
        self.post_norm_block_ids = post_norm_block_ids
        if post_norm_block_ids is not None:
            self.post_norms = nn.ModuleList([build_norm_layer(channels, "LN", eps=1e-6) for _ in post_norm_block_ids])
        self.downsample = DownsampleLayer(channels=channels, norm_layer=norm_layer) if downsample else None

    def forward(self, x, return_wo_downsample=False):
        for i, blk in enumerate(self.blocks):
            x = blk(x)
            if self.post_norm_block_ids is not None and i in self.post_norm_block_ids:
                x = _apply_ln(self.post_norms[self.post_norm_block_ids.index(i)], x)
        if not self.post_norm or self.center_feature_scale:
            x = _apply_ln(self.norm, x)
        x_ = x
        if self.downsample is not None:
            x = self.downsample(x)
        return (x, x_) if return_wo_downsample else x


class B200InternImage(nn.Module):
    """`InternImage` (gd.py:4978-5152).  forward(x[B,3,H,W]) -> list of level maps.  `channels_last_out=True` (default
    inside the H100 GDINO stage) returns [B, h, w, C] maps flagged `_b200_nhwc`; False returns the reference's
    contiguous NCHW maps."""

    def __init__(self, core_op="DCNv3", channels=64, depths=(3, 4, 18, 5), groups=(3, 6, 12, 24), mlp_ratio=4.,
                 drop_rate=0., drop_path_rate=0.2, drop_path_type="linear", act_layer="GELU", norm_layer="LN",
                 layer_scale=None, offset_scale=1.0, post_norm=False, with_cp=False, dw_kernel_size=None,
                 level2_post_norm=False, level2_post_norm_block_ids=None, res_post_norm=False,
                 center_feature_scale=False, out_indices=(0, 1, 2, 3), init_cfg=None, channels_last_out=True, **kwargs):
        super().__init__()
        if core_op not in ("DCNv3", "DCNv3_pytorch"):
            raise NotImplementedError(f"core_op={core_op}")
        depths, groups = list(depths), list(groups)
        self.core_op, self.num_levels, self.depths, self.channels_first_stage = core_op, len(depths), depths, channels
        self.num_features = [int(channels * 2 ** i) for i in range(self.num_levels)]
        self.channels = list(self.num_features)          # what the GDINO conv-encoder shell reads
        self.post_norm, self.mlp_ratio, self.out_indices = post_norm, mlp_ratio, tuple(out_indices)
        self.channels_last_out = channels_last_out
        self.patch_embed = StemLayer(in_chans=3, out_chans=channels, act_layer=act_layer, norm_layer=norm_layer)
        self.pos_drop = nn.Dropout(p=drop_rate)
        self.levels = nn.ModuleList()
        for i in range(self.num_levels):
            ids = level2_post_norm_block_ids if level2_post_norm and i == 2 else None
            self.levels.append(InternImageBlock(
                core_op=DCNv3, channels=int(channels * 2 ** i), depth=depths[i], groups=groups[i],
                mlp_ratio=mlp_ratio, drop=drop_rate, act_layer=act_layer, norm_layer=norm_layer, post_norm=post_norm,
                downsample=(i < self.num_levels - 1), layer_scale=layer_scale, offset_scale=offset_scale,
                dw_kernel_size=dw_kernel_size, post_norm_block_ids=ids, res_post_norm=res_post_norm,
                center_feature_scale=center_feature_scale))
        self.num_layers = len(depths)

    @torch.no_grad()
    def forward(self, x):
        x = self.patch_embed(x)
        seq_out = []
        for level_idx, level in enumerate(self.levels):
            x, x_ = level(x, return_wo_downsample=True)
            if level_idx in self.out_indices:
                if self.channels_last_out:
                    x_ = x_.contiguous()
                    x_._b200_nhwc = True
                    seq_out.append(x_)
                else:
                    seq_out.append(x_.permute(0, 3, 1, 2).contiguous())
        return seq_out


INTERNIMAGE_H = dict(core_op="DCNv3", channels=320, depths=[6, 6, 32, 6], groups=[10, 20, 40, 80], mlp_ratio=4.,
                     drop_path_rate=0., norm_layer="LN", layer_scale=None, offset_scale=1.0, post_norm=False,
                     dw_kernel_size=5, res_post_norm=True, level2_post_norm=True,
                     level2_post_norm_block_ids=[5, 11, 17, 23, 29], center_feature_scale=True, with_cp=True,
                     out_indices=(0, 1, 2, 3), init_cfg=None)


def build_internimage_h(cfg_hf=None, **kw):
    """`build_internimage_h` (gd.py:5154-5184): the InternImage-H preset, overridable by a dict."""
    cfg = dict(INTERNIMAGE_H)
    if isinstance(cfg_hf, dict):
        cfg.update(cfg_hf)
    cfg.pop("load_path", None)
    cfg.update(kw)
    backbone = B200InternImage(**cfg)
    # the reference pins the neck's input widths to the H preset whatever the overrides say (gd.py:5183)
    backbone.num_features = [320, 640, 1280, 2560]
    backbone.channels = list(backbone.num_features)
    return backbone
