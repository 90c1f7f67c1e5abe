"""H100-native region encoder (SURVEY.md 8f rank 4): drop-in for `RegionEncoder`
(visionllmv2/model/region_encoder.py:66-145; built at modeling_visionllmv2.py:247-252 with mask_pool_type='grid_sample',
called at :687 with the [n_regions, 3, H, W] images, the [n_regions, 1, H, W] 0/1 region masks and the last three ViT
hidden states).  Same constructor, parameter names (`mask_embedding.{0,1,3,4,6}`, `up_dim`, `region_query`,
`region_attn`) and forward contract `forward(images, masks, image_features) -> [n_regions, out_dim]`.

On our kernels, channels-last:
  mask_embedding   the two patchify convs (k7 s7, k2 s2) and the 1x1 conv are plain GEMMs over non-overlapping patches
                   (weights used in their native [Cout, Cin*k*k] order, K zero-padded to a 16-byte pitch);
                   LayerNorm2d (LN over channels) + GELU is ONE row-kernel pass each.
  'mean'           the reference's bilinear-resized mask (same torch op => same binary mask) and a masked mean.
  'cross_attn'     nn.MultiheadAttention with one learnable query: packed in_proj GEMMs + fused attention + out_proj.
  'grid_sample'    `point_sample` (= bilinear grid_sample, align_corners=False, zero padding, [0,1] coordinates) IS the
                   MSDA sampling rule with one level, so the up-to-2304 sampled points of a region are pooled by the
                   MSDA kernel (16 points per query, weights 1 for real points and 0 for padding) and a sum.
The sampler (`rand_sample`: torch.multinomial over the region's pixels, region_encoder.py:50-64) is random by design;
it is restated below for production use (one draw per feature level and region, like the reference), and
`forward(..., sample_points=[level][region] -> [n, 3])` takes the points explicitly so parity tests can feed the
reference's own draw.  The reference accumulates `masks_out` across the feature levels (and, in
'mean' mode, keeps the mask product) -- reproduced as is.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import msda as msda_ext
from . import ops


class LayerNorm2d(nn.Module):
    """Parameter holder of the reference's LayerNorm2d (region_encoder.py:9-22): LN over the channel axis."""

    def __init__(self, num_channels, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(num_channels))
        self.bias = nn.Parameter(torch.zeros(num_channels))
        self.eps = eps


def rand_sample(x, divisor, max_len):
    """region_encoder.py:50-64, restated: up to `max_len` of the region's non-zero pixels, drawn without replacement
    with equal probability per mask id; returns [n, 3] rows (mask id, y / H, x / W)."""
    nz = x.nonzero()
    if len(nz) == 0:
        return nz
    pts = (nz / divisor).t()
    ids = pts[0].unique().long()
    probs = torch.zeros_like(pts[0])
    for idx in ids:
        probs[pts[0] == idx] = 1. / (len(ids) * ((pts[0:1] == idx).sum()))
    indices = torch.multinomial(probs, num_samples=min(max_len, len(probs)), replacement=False).sort()[0]
    return pts[:, indices].t()


POOL_GROUP = 16                                  # points per MSDA query of the pooling


def point_table(points, device):
    """[region] -> [n_i, 3] (id, y, x in [0,1]) points -> the pooling's packed table: loc [B, n_pad, 2] fp32 (x, y) and
    wgt [B, n_pad] fp32 (1 for a point, 0 for padding), n_pad the longest list rounded up to a query group of 16 (at
    least one group).  The forward pools through it and the training backward transposes the same table."""
    B, P = len(points), POOL_GROUP
    n_max = max([len(p) for p in points] + [1])
    Lq = (n_max + P - 1) // P
    loc = torch.zeros(B, Lq * P, 2, dtype=torch.float32, device=device)
    wgt = torch.zeros(B, Lq * P, dtype=torch.float32, device=device)
    for i, p in enumerate(points):
        n = len(p)
        if n:
            loc[i, :n] = p[:, -2:].flip(-1).float()                                         # (x, y)
            wgt[i, :n] = 1.0
    return loc, wgt


def _patch_rows(x, k):
    """[B, H, W, C] channels-last -> [B*(H/k)*(W/k), C*k*k] rows in the (c, dy, dx) order of a Conv2d weight."""
    B, Hh, W, C = x.shape
    h, w = Hh // k, W // k
    x = x[:, :h * k, :w * k].reshape(B, h, k, w, k, C).permute(0, 1, 3, 5, 2, 4)
    return x.reshape(B * h * w, C * k * k), h, w


class B200RegionEncoder(nn.Module):
    def __init__(self, hidden_dim, embed_dim, out_dim, patch_size=14, mask_pool_type="mean"):
        super().__init__()
        assert patch_size % 2 == 0
        kernel_size = patch_size // 2
        self.patch_size = patch_size
        self.mask_embedding = nn.Sequential(
            nn.Conv2d(4, hidden_dim // 4, kernel_size=kernel_size, stride=kernel_size),
            LayerNorm2d(hidden_dim // 4),
            nn.GELU(),
            nn.Conv2d(hidden_dim // 4, hidden_dim, kernel_size=2, stride=2),
            LayerNorm2d(hidden_dim),
            nn.GELU(),
            nn.Conv2d(hidden_dim, embed_dim, kernel_size=1),
        )
        self.mask_pool_type = mask_pool_type
        assert mask_pool_type in ["mean", "cross_attn", "grid_sample"]
        if mask_pool_type == "cross_attn":
            self.region_query = nn.Embedding(1, embed_dim)
            self.region_attn = nn.MultiheadAttention(embed_dim=embed_dim, num_heads=8, dropout=0., batch_first=True)
        elif mask_pool_type == "grid_sample":
            self.num_points = 2304
        self.up_dim = nn.Linear(embed_dim, out_dim)
        self._w = {}

    # ---- pieces ---------------------------------------------------------------------------------------------
    def _conv_rows(self, rows, conv, tag):
        """rows [M, Cin*k*k] -> [M, Cout]; the weight keeps its native order, K padded to a multiple of 8."""
        K = rows.shape[1]
        Kp = (K + 7) // 8 * 8
        key = (tag, conv.weight.data_ptr(), conv.weight._version, rows.dtype)
        if self._w.get(tag, (None,))[0] != key:
            w = conv.weight.detach().reshape(conv.out_channels, K).to(rows.dtype)
            self._w[tag] = (key, F.pad(w, (0, Kp - K)).contiguous() if Kp != K else w.contiguous())
        if Kp != K:
            rows = F.pad(rows, (0, Kp - K))
        return ops.linear(rows.contiguous(), self._w[tag][1], bias=conv.bias.detach().to(rows.dtype))

    def embed_masks(self, images, masks):
        """mask_embedding on cat([images, masks], 1): -> channels-last [B, h, w, embed_dim]."""
        me = self.mask_embedding
        x = torch.cat([images, masks.to(images.dtype)], dim=1).permute(0, 2, 3, 1)           # [B, H, W, 4]
        B = x.shape[0]
        rows, h, w = _patch_rows(x, me[0].kernel_size[0])
        y = self._conv_rows(rows, me[0], "c0")
        y = ops.layernorm(y, me[1].weight, me[1].bias, me[1].eps, gelu=True)
        rows, h, w = _patch_rows(y.view(B, h, w, -1), 2)
        y = self._conv_rows(rows, me[3], "c3")
        y = ops.layernorm(y, me[4].weight, me[4].bias, me[4].eps, gelu=True)
        y = self._conv_rows(y, me[6], "c6")
        return y.view(B, h, w, -1)

    def draw_points(self, masks, levels):
        """The production draw: `rand_sample` per feature level and region, in the order the reference draws them
        (:123-125) -> [level][region] -> [n, 3]."""
        ori_h, ori_w = masks.shape[-2:]
        divisor = torch.tensor([1, ori_h, ori_w], device=masks.device)[None,]
        return [[rand_sample(m, divisor, self.num_points) for m in masks] for _ in range(levels)]

    def _pool_points(self, feat, loc, wgt):
        """feat [B, h, w, C]; the point table of `point_table` -> masked mean of the bilinear samples."""
        B, h, w, C = feat.shape
        D = 32
        if C % D:
            raise NotImplementedError("grid_sample pooling needs embed_dim % 32 == 0")
        M, P = C // D, POOL_GROUP
        Lq = loc.shape[1] // P
        shapes = msda_ext.attach_host_shapes(torch.tensor([[h, w]], dtype=torch.int64, device=feat.device), [(h, w)])
        lsi = torch.zeros(1, dtype=torch.int64, device=feat.device)
        value = feat.float().reshape(B, h * w, M, D).contiguous()
        loc6 = loc.view(B, Lq, 1, 1, P, 2).expand(B, Lq, M, 1, P, 2).contiguous()
        w5 = wgt.view(B, Lq, 1, 1, P).expand(B, Lq, M, 1, P).contiguous()
        out = msda_ext.ms_deform_attn_forward(value, shapes, lsi, loc6, w5, B)              # [B, Lq, C]
        cnt = wgt.sum(1, keepdim=True)
        return (out.sum(1) / cnt).nan_to_num().to(feat.dtype)

    def _pool_cross_attn(self, feat):
        B, h, w, C = feat.shape
        at = self.region_attn
        Wq, Wk, Wv = at.in_proj_weight.detach().chunk(3, 0)
        bq, bk, bv = at.in_proj_bias.detach().chunk(3, 0)
        dt = feat.dtype
        kv = feat.reshape(B, h * w, C)
        q = ops.linear(self.region_query.weight.detach().to(dt).expand(B, C).contiguous(), Wq.to(dt).contiguous(),
                       bias=bq.to(dt).contiguous())
        k = ops.linear(kv, Wk.to(dt).contiguous(), bias=bk.to(dt).contiguous())
        v = ops.linear(kv, Wv.to(dt).contiguous(), bias=bv.to(dt).contiguous())
        H = at.num_heads
        ctx = ops.attention(q.view(B, 1, H, C // H), k.view(B, h * w, H, C // H), v.view(B, h * w, H, C // H))
        return ops.linear(ctx.reshape(B, C), at.out_proj.weight.detach().to(dt), bias=at.out_proj.bias.detach().to(dt))

    # ---- forward ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, images, masks, image_features, sample_points=None):
        assert images.shape[-2:] == masks.shape[-2:]
        masks = masks.to(images.dtype)
        masks_out = self.embed_masks(images, masks)                                           # [B, h, w, E]
        bs, h, w, _ = masks_out.shape
        outs = []
        for level, feats in enumerate(image_features):
            f = feats.reshape(bs, h, w, -1) if feats.dim() == 3 else feats.permute(0, 2, 3, 1)
            assert masks_out.shape[1:3] == f.shape[1:3]
            masks_out = masks_out + f.to(masks_out.dtype)
            if self.mask_pool_type == "mean":
                binary = F.interpolate(masks.float(), size=(h, w), mode="bilinear", align_corners=False) > 0.5
                masks_out = masks_out * binary.permute(0, 2, 3, 1)
                out = masks_out.mean((1, 2))
            elif self.mask_pool_type == "cross_attn":
                out = self._pool_cross_attn(masks_out)
            else:
                if sample_points is not None:
                    pts = sample_points[level]
                else:                                   # a fresh draw per level, like the reference (:123-125)
                    pts = self.draw_points(masks, 1)[0]
                out = self._pool_points(masks_out, *point_table(pts, masks_out.device))
            outs.append(ops.linear(out.contiguous(), self.up_dim.weight, bias=self.up_dim.bias))
        return torch.stack(outs).mean(dim=0)
