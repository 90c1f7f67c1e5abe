"""The Grounding-DINO region / mask decoder as ONE module with the reference's constructor, parameter names and
test-time forward (SURVEY 8a rows a12-a20): `OVGroundingDinoForObjectDetection.forward_test`
(grounding_dino/modeling_ov_grounding_dino_mask_dn.py:3124-3210) over `OVGroundingDinoModel.forward` (:2283-2600),
`GroundingDinoEncoder.forward` (:1575-1722) and `GroundingDinoDecoder.forward` (:1792-1981).

What runs where:
  backbone (a13)            HF `AutoBackbone` (Swin) exactly as the reference builds it (:471-504) -- third-party
                            torch code on the GPU, or `visionllm_b200.swin.B200SwinBackbone` (same state dict) when
                            passed in.  Everything after it is ours.
  neck (a14)                1x1 / 3x3-stride-2 projections as wgmma GEMMs over channels-last rows + the GroupNorm
                            kernel (csrc/groupnorm.cu); sine position embedding, masks, `spatial_shapes`,
                            `level_start_index`, `valid_ratios` with the reference's own integer / fp32 arithmetic.
  encoder / decoder         visionllm_b200.gdino layers (MSDA kernel, fused attention, GEMM epilogues).
  mask-feature FPN (a20)    lateral 1x1 + GN, bilinear upsample-add, 3x3 + GN + ReLU, 1x1 -- GEMMs + GroupNorm kernel.
  two-stage selection (a18) visionllm_b200.gdino_heads (torch.topk for index parity).
  heads (a20)               bbox MLP + inverse-sigmoid(ref), contrastive logits, mask einsum as GEMM.

Activations stay channels-last ([B, H*W, C] rows) from the backbone output to the encoder input, so no
flatten(2).transpose(1, 2) copies (:2418-2422) are needed.  Inference only: training (contrastive DN, losses) is out
of scope and raises.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import gdino_heads as H
from . import msda, ops
from .gdino import GroundingDinoDecoderLayer, GroundingDinoEncoderLayer


def inverse_sigmoid(x, eps=1e-5):
    """gd.py:3722-3727 (clamp to [0,1], then log(max(x,eps)/max(1-x,eps)))."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


def generate_masks_with_text_query_masks(text_query_masks):
    """gd.py:2025-2042: block of ones over the valid prefix + identity, and 0..n-1 position ids."""
    B, T = text_query_masks.shape
    dev = text_query_masks.device
    n = text_query_masks.sum(1)                                           # valid count per row
    ar = torch.arange(T, device=dev)
    pre = ar[None, :] < n[:, None]
    mask = (pre[:, :, None] & pre[:, None, :]) | torch.eye(T, dtype=torch.bool, device=dev)[None]
    pos = torch.where(pre, ar[None, :].expand(B, -1), torch.zeros((), dtype=torch.long, device=dev))
    return mask, pos


class GroundingDinoSinePositionEmbedding(nn.Module):
    """gd.py:529-564, producing channels-last [B, H, W, 2*embedding_dim] (the reference permutes to NCHW and the
    caller transposes back, :2420)."""

    def __init__(self, embedding_dim=64, temperature=10000, normalize=False, scale=None):
        super().__init__()
        if scale is not None and normalize is False:
            raise ValueError("normalize should be True if scale is passed")
        self.embedding_dim, self.temperature, self.normalize = embedding_dim, temperature, normalize
        self.scale = 2 * math.pi if scale is None else scale

    @torch.no_grad()
    def embeds(self, pixel_mask):
        """(y_embed, x_embed) fp32 [B, H, W]: the normalised cumulative coordinates (gd.py:545-551)."""
        y_embed = pixel_mask.cumsum(1, dtype=torch.float32)
        x_embed = pixel_mask.cumsum(2, dtype=torch.float32)
        if self.normalize:
            eps = 1e-6
            y_embed = y_embed / (y_embed[:, -1:, :] + eps) * self.scale
            x_embed = x_embed / (x_embed[:, :, -1:] + eps) * self.scale
        return y_embed, x_embed

    def dim_t(self, device):
        """temperature ** (2 * (d // 2) / embedding_dim), fp32 [embedding_dim] (gd.py:553-554), cached per device."""
        cache = self.__dict__.setdefault("_dim_t", {})
        if str(device) not in cache:
            d = torch.arange(self.embedding_dim, dtype=torch.float32, device=device)
            cache[str(device)] = self.temperature ** (2 * torch.div(d, 2, rounding_mode="floor") / self.embedding_dim)
        return cache[str(device)]

    @torch.no_grad()
    def forward(self, pixel_mask):
        y_embed, x_embed = self.embeds(pixel_mask)
        dim_t = self.dim_t(pixel_mask.device)
        pos_x = x_embed[:, :, :, None] / dim_t
        pos_y = y_embed[:, :, :, None] / dim_t
        pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
        pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
        return torch.cat((pos_y, pos_x), dim=3)


def conv_rows(x, conv, prepadded=False, keep_grid=False):
    """Conv2d over a channels-last map x [B, H, W, Cin] as ONE GEMM on [B*Ho*Wo, kh*kw*Cin] rows (tap-major K, the
    weight repacked to match); returns ([B, Ho*Wo, Cout], Ho, Wo).  1x1 convs read the map in place."""
    kh, kw = conv.kernel_size
    s, p = conv.stride[0], conv.padding[0]
    implicit = s == 1 and kh == kw and kh > 1 and (kw * x.shape[3]) % 64 == 0 and conv.padding[0] == conv.padding[1]
    if prepadded and not implicit:
        x = x[:, p:x.shape[1] - p, p:x.shape[2] - p]                               # not the implicit-GEMM form: drop the border again
    B, Hh, W, C = x.shape
    if (kh, kw, s, p) == (1, 1, 1, 0):
        rows, Ho, Wo = x.reshape(B, Hh * W, C), Hh, W
    elif implicit:
        # implicit GEMM over the zero-padded map: no [B*Ho*Wo, kh*kw*C] im2col buffer
        w = conv.weight.permute(0, 2, 3, 1).reshape(conv.out_channels, -1).contiguous()
        y = ops.conv2d_s1_rows(x, w, conv.bias, kh, p, prepadded=prepadded)
        if keep_grid:                                                                # the valid corner of the padded grid, in place
            return y, y.shape[1], y.shape[2]
        return y.reshape(B, y.shape[1] * y.shape[2], conv.out_channels), y.shape[1], y.shape[2]
    else:
        Ho, Wo = (Hh + 2 * p - kh) // s + 1, (W + 2 * p - kw) // s + 1
        xp = F.pad(x, (0, 0, p, p, p, p))
        taps = [xp[:, dy:dy + s * (Ho - 1) + 1:s, dx:dx + s * (Wo - 1) + 1:s, :] for dy in range(kh) for dx in range(kw)]
        rows = torch.cat(taps, -1).reshape(B, Ho * Wo, kh * kw * C)
    w = conv.weight.permute(0, 2, 3, 1).reshape(conv.out_channels, -1)
    if kh * kw > 1 or not w.is_contiguous():
        w = w.contiguous()
    return ops.linear(rows.contiguous(), w, bias=conv.bias), Ho, Wo


class NormConv2d(nn.Conv2d):
    """detectron2.layers.Conv2d(norm=GroupNorm(32, C)[, activation=relu]) as the mask FPN uses it (gd.py:2126-2151):
    parameters `weight`, `norm.weight`, `norm.bias` (no conv bias when a norm is attached)."""

    def __init__(self, cin, cout, kernel_size, padding=0, relu=False):
        super().__init__(cin, cout, kernel_size, padding=padding, bias=False)
        self.norm = nn.GroupNorm(32, cout)
        self.relu = relu

    @torch.no_grad()
    def rows(self, x, prepadded=False):
        """prepadded: x is the zero-bordered map `ops.upsample_add_nhwc(..., pad=)` wrote.  The GroupNorm reads the 3x3
        convolution's output corner of the padded grid in place (no compaction copy)."""
        y, Ho, Wo = conv_rows(x, self, prepadded=prepadded, keep_grid=True)
        return ops.groupnorm_nhwc(y, self.norm.weight, self.norm.bias, self.norm.num_groups, self.norm.eps, relu=self.relu), Ho, Wo


class _ConvEncoder(nn.Module):
    """Key-compatible shell of GroundingDinoConvEncoder (gd.py:471-504): `.model` is the HF backbone."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.intermediate_channel_sizes = list(model.channels)


class _ConvModel(nn.Module):
    """GroundingDinoConvModel (gd.py:508-526): backbone + position embedding (no parameters of its own)."""

    def __init__(self, conv_encoder, position_embedding):
        super().__init__()
        self.conv_encoder = conv_encoder
        self.position_embedding = position_embedding


class _Encoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layers = nn.ModuleList([GroundingDinoEncoderLayer(config) for _ in range(config.encoder_layers)])
        for layer in self.layers:                              # this stage discards the encoder's attention maps (forward_test)
            layer.deformable_layer.self_attn.need_weights = False

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        """gd.py:1577-1605."""
        refs = []
        for level, (height, width) in enumerate(msda.host_shape_list(spatial_shapes)):
            ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, height - 0.5, height, dtype=torch.float32, device=device),
                                          torch.linspace(0.5, width - 0.5, width, dtype=torch.float32, device=device),
                                          indexing="ij")
            ref_y = ref_y.reshape(-1)[None] / (valid_ratios[:, None, level, 1] * height)
            ref_x = ref_x.reshape(-1)[None] / (valid_ratios[:, None, level, 0] * width)
            refs.append(torch.stack((ref_x, ref_y), -1))
        reference_points = torch.cat(refs, 1)
        return reference_points[:, :, None] * valid_ratios[:, None]


class _Decoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layer_norm = nn.LayerNorm(config.d_model)
        self.layers = nn.ModuleList([GroundingDinoDecoderLayer(config) for _ in range(config.decoder_layers)])
        self.reference_points_head = H.GroundingDinoMLPPredictionHead(config.query_dim // 2 * config.d_model,
                                                                      config.d_model, config.d_model, 2)
        self.bbox_embed = None
        self.d_model = config.d_model

    def _dim_t(self, device):
        cache = self.__dict__.setdefault("_dim_t_cache", {})
        if str(device) not in cache:
            num_pos_feats = self.d_model // 2
            d = torch.arange(num_pos_feats, dtype=torch.float32, device=device)
            cache[str(device)] = 10000 ** (2 * torch.div(d, 2, rounding_mode="floor") / num_pos_feats)
        return cache[str(device)]

    def proposal_pos_embed_rows(self, proposals, out_dtype):
        """`get_proposal_pos_embed(proposals).to(out_dtype)` for fp32 CUDA proposals [B, Q, 2 | 4] whose last-axis elements are
        `proposals.stride(1)` apart per query (e.g. `ref_in[:, :, 0, :]`): ONE launch of csrc/posembed.cu instead of ~26."""
        B, Q, k = proposals.shape
        if (not proposals.is_cuda or proposals.dtype != torch.float32 or out_dtype not in (torch.float32, torch.bfloat16)
                or proposals.stride(2) != 1 or proposals.stride(0) != Q * proposals.stride(1) or k not in (2, 4)):
            return self.get_proposal_pos_embed(proposals).to(out_dtype)
        order = (1, 0) if k == 2 else (1, 0, 2, 3)
        feats = [proposals[:, :, c] for c in order]
        out = ops.sine_embed(feats, proposals.stride(1), self._dim_t(proposals.device), B * Q, pre_scale=2 * math.pi,
                             out_dtype=out_dtype)
        return out.view(B, Q, -1)

    def get_proposal_pos_embed(self, proposals):
        """gd.py:1755-1790: (y, x[, w, h]) sin/cos features, fp32."""
        num_pos_feats = self.d_model // 2
        dim_t = self._dim_t(proposals.device)

        def feat(col):
            e = (proposals[:, :, col] * (2 * math.pi))[:, :, None] / dim_t
            return torch.stack((e[:, :, 0::2].sin(), e[:, :, 1::2].cos()), dim=3).flatten(2)

        if proposals.size(-1) == 2:
            return torch.cat((feat(1), feat(0)), dim=2)
        if proposals.size(-1) == 4:
            return torch.cat((feat(1), feat(0), feat(2), feat(3)), dim=2)
        raise ValueError("Unknown proposals shape(-1):{}".format(proposals.size(-1)))


class B200GroundingDinoModel(nn.Module):
    def __init__(self, config, backbone_model=None):
        super().__init__()
        self.config = config
        if backbone_model is None:
            bc = config.backbone_config
            mtype = bc.get("model_type") if isinstance(bc, dict) else getattr(bc, "model_type", None)
            if mtype == "internimage-H":                 # gd.py:2073-2074 / 5186-5195: a plain dict of overrides
                from .internimage import build_internimage_h
                backbone_model = build_internimage_h({k: v for k, v in bc.items() if k != "model_type"})
            elif mtype == "swin":
                from transformers import AutoBackbone
                backbone_model = AutoBackbone.from_config(bc)
            else:
                raise NotImplementedError(f"backbone model_type={mtype!r} (the reference wires 'swin' and 'internimage-H')")
        enc = _ConvEncoder(backbone_model)
        self.backbone = _ConvModel(enc, GroundingDinoSinePositionEmbedding(
            config.d_model // 2, config.positional_embedding_temperature, normalize=True))
        if config.position_embedding_type != "sine":
            raise NotImplementedError("learned position embedding")
        chans = enc.intermediate_channel_sizes
        d = config.d_model
        if config.num_feature_levels <= 1:
            raise NotImplementedError("single-level neck")
        proj, cin = [], None
        for cin in chans[-3:]:
            proj.append(nn.Sequential(nn.Conv2d(cin, d, kernel_size=1), nn.GroupNorm(32, d)))
        for _ in range(config.num_feature_levels - len(chans[-3:])):
            proj.append(nn.Sequential(nn.Conv2d(cin, d, kernel_size=3, stride=2, padding=1), nn.GroupNorm(32, d)))
            cin = d
        self.input_proj_vision = nn.ModuleList(proj)
        self.num_fpn_levels = max(config.num_feature_levels - len(chans[-3:]), 1)
        if config.norm != "GN":
            raise NotImplementedError("mask FPN norm other than GN")
        self.mask_features = nn.Conv2d(d, config.mask_dim, kernel_size=1)
        self.lateral_convs = nn.ModuleList([NormConv2d(c, d, 1) for c in chans[:self.num_fpn_levels]])
        self.output_convs = nn.ModuleList([NormConv2d(d, d, 3, padding=1, relu=True) for _ in chans[:self.num_fpn_levels]])
        if config.embedding_init_target or not config.two_stage:
            self.query_position_embeddings = nn.Embedding(config.num_queries, d)
        self.mask_embed = H.GroundingDinoMLPPredictionHead(d, d, config.mask_dim, 3)
        self.encoder = _Encoder(config)
        self.decoder = _Decoder(config)
        self.level_embed = nn.Parameter(torch.zeros(config.num_feature_levels, d))
        if not config.two_stage:
            raise NotImplementedError("single-stage (learned reference points) variant")
        self.enc_output = nn.Linear(d, d)
        self.enc_output_norm = nn.LayerNorm(d)
        if config.two_stage_bbox_embed_share:
            raise NotImplementedError("two_stage_bbox_embed_share")
        self.encoder_output_bbox_embed = H.GroundingDinoMLPPredictionHead(d, d, 4, 3)
        self.encoder_output_class_embed = H.GroundingDinoContrastiveEmbedding(config)
        self._shape_cache = {}

    @staticmethod
    def get_valid_ratio(mask):
        """gd.py:2202-2211."""
        _, height, width = mask.shape
        valid_height = torch.sum(mask[:, :, 0], 1)
        valid_width = torch.sum(mask[:, 0, :], 1)
        return torch.stack([valid_width.float() / width, valid_height.float() / height], -1)

    @torch.no_grad()
    def backbone_features(self, pixel_values):
        """[B,3,H,W] -> list of channels-last maps [B, h, w, C_l] (strides 4/8/16/32)."""
        out = self.backbone.conv_encoder.model(pixel_values)
        maps = out.feature_maps if hasattr(out, "feature_maps") else out
        return [m if getattr(m, "_b200_nhwc", False) else m.permute(0, 2, 3, 1).contiguous() for m in maps]

    def _shape_tensors(self, shapes, device):
        """int64 `spatial_shapes` [L, 2] and `level_start_index` [L] (exclusive cumsum, gd.py:2434-2437); built once
        per pyramid (a host->device copy) with the host list attached, so a forward has no sync."""
        key = (shapes, str(device))
        if key not in self._shape_cache:
            ss = msda.attach_host_shapes(torch.as_tensor(shapes, dtype=torch.long, device=device), shapes)
            lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
            self._shape_cache[key] = (ss, lsi)
        return self._shape_cache[key]

    @torch.no_grad()
    def neck(self, feats, pixel_mask):
        """Input projections + flatten (gd.py:2388-2439).  feats: channels-last backbone maps (all 4 stages)."""
        dtype = feats[0].dtype
        pm = pixel_mask[None].float()
        pos_embed = self.backbone.position_embedding
        sources, masks, poss, shapes = [], [], [], []
        for level, f in enumerate(feats[1:]):
            seq = self.input_proj_vision[level]
            y, Ho, Wo = conv_rows(f, seq[0])
            sources.append(ops.groupnorm_nhwc(y, seq[1].weight, seq[1].bias, seq[1].num_groups, seq[1].eps))
            masks.append(F.interpolate(pm, size=(Ho, Wo)).to(torch.bool)[0])
            shapes.append((Ho, Wo))
        n_in = len(sources)
        for level in range(n_in, self.config.num_feature_levels):
            seq = self.input_proj_vision[level]
            src = feats[-1] if level == n_in else sources[-1].view(feats[0].shape[0], *shapes[-1], -1)
            y, Ho, Wo = conv_rows(src, seq[0])
            sources.append(ops.groupnorm_nhwc(y, seq[1].weight, seq[1].bias, seq[1].num_groups, seq[1].eps))
            masks.append(F.interpolate(pm, size=(Ho, Wo)).to(torch.bool)[0])
            shapes.append((Ho, Wo))
        source_flatten = torch.cat(sources, 1)
        mask_flatten = torch.cat([m.flatten(1) for m in masks], 1)
        if (dtype == torch.bfloat16 and source_flatten.is_cuda and self.level_embed.dtype == torch.bfloat16
                and isinstance(pos_embed, GroundingDinoSinePositionEmbedding)):
            # sine position embedding -> bf16 -> + level embedding, one launch per level, written straight into its slab of
            # the flattened buffer (csrc/posembed.cu: the reference's fp32 arithmetic, element for element)
            lvl_pos_embed_flatten = torch.empty_like(source_flatten)
            dim_t, off = pos_embed.dim_t(source_flatten.device), 0
            for level, m in enumerate(masks):
                y_embed, x_embed = pos_embed.embeds(m)
                n = m.shape[1] * m.shape[2]
                ops.sine_embed([y_embed.contiguous(), x_embed.contiguous()], 1, dim_t, m.shape[0] * n,
                               out=lvl_pos_embed_flatten[:, off:off + n], add_row=self.level_embed[level].contiguous())
                off += n
        else:
            for level, m in enumerate(masks):
                pos = pos_embed(m).to(dtype).flatten(1, 2)                                # [B, HW, d]
                poss.append(pos + self.level_embed[level].view(1, 1, -1))
            lvl_pos_embed_flatten = torch.cat(poss, 1)
        spatial_shapes, level_start_index = self._shape_tensors(tuple(shapes), source_flatten.device)
        valid_ratios = torch.stack([self.get_valid_ratio(m) for m in masks], 1).float()
        return source_flatten, mask_flatten, lvl_pos_embed_flatten, spatial_shapes, level_start_index, valid_ratios

    @torch.no_grad()
    def build_mask_features(self, feats, enc_vision, spatial_shapes):
        """gd.py:2470-2497 for num_fpn_levels == 1: returns (rows [B, H*W, mask_dim], H, W)."""
        B = enc_vision.shape[0]
        H0, W0 = msda.host_shape_list(spatial_shapes)[0]
        top = enc_vision[:, :H0 * W0].reshape(B, H0, W0, -1)                              # level-0 slab, channels-last
        for idx in range(self.num_fpn_levels):
            cur, Hc, Wc = self.lateral_convs[idx].rows(feats[idx])
            oc = self.output_convs[idx]
            pad = oc.padding[0] if oc.padding[0] == oc.padding[1] and oc.stride[0] == 1 else 0
            # lateral + bilinear(top) in one pass, written straight into the output convolution's zero-padded input; `top` (the
            # level-0 slab of the flattened encoder output at idx 0) is read in place through its batch pitch
            y = ops.upsample_add_nhwc(top, cur.view(B, Hc, Wc, -1), pad=pad)
            top, Hc, Wc = oc.rows(y, prepadded=pad > 0)
            top = top.view(B, Hc, Wc, -1)
        mf, Hm, Wm = conv_rows(top, self.mask_features)
        return mf, Hm, Wm

    @torch.no_grad()
    def forward(self, pixel_values, pixel_mask=None, text_query=None, text_query_masks=None):
        cfg = self.config
        tsa, position_ids = generate_masks_with_text_query_masks(text_query_masks)
        text_token_mask = text_query_masks.bool()
        if tsa.shape[1] > cfg.max_text_len:
            L = cfg.max_text_len
            tsa, position_ids, text_token_mask = tsa[:, :L, :L], position_ids[:, :L], text_token_mask[:, :L]
        B, _, height, width = pixel_values.shape
        if pixel_mask is None:
            pixel_mask = torch.ones((B, height, width), dtype=torch.long, device=pixel_values.device)
        feats = self.backbone_features(pixel_values)
        src, mask_flatten, pos, spatial_shapes, lsi, valid_ratios = self.neck(feats, pixel_mask)
        # encoder (gd.py:1650-1722); key_padding_mask convention: True = padding
        kpm = ~mask_flatten
        ref2 = _Encoder.get_reference_points(spatial_shapes, valid_ratios, src.device)
        v, t = src, text_query
        # the text position embedding depends on position_ids only: computed once, not once per layer (gd.py:1131-1150 recomputes
        # the same tensor in every layer)
        tpos = (self.encoder.layers[0].get_text_position_embeddings(t, None, position_ids).to(src.dtype)
                if len(self.encoder.layers) else None)
        text_pad = ~text_token_mask
        for layer in self.encoder.layers:
            (v, t), _ = layer(vision_features=v, vision_position_embedding=pos, spatial_shapes=spatial_shapes,
                              level_start_index=lsi, key_padding_mask=kpm, reference_points=ref2, text_features=t,
                              text_attention_mask=text_pad, text_position_embedding=tpos,
                              text_self_attention_masks=tsa, text_position_ids=None)
        mask_features = self.build_mask_features(feats, v, spatial_shapes)
        # two-stage query selection (gd.py:2503-2545)
        oq, proposals = H.gen_encoder_output_proposals(self.enc_output, self.enc_output_norm, v, kpm, spatial_shapes)
        enc_class = self.encoder_output_class_embed(oq, t, text_token_mask)
        enc_coord = self.encoder_output_bbox_embed(oq) + proposals
        topk_idx, reference_points, enc_topk_coords, enc_topk_class, target_undetach = H.select_topk_proposals(
            enc_class, enc_coord, oq, cfg.num_queries)
        if cfg.embedding_init_target:
            target = self.query_position_embeddings.weight.unsqueeze(0).repeat(B, 1, 1)
        else:
            target = target_undetach
        init_reference_points = reference_points
        # decoder (gd.py:1870-1981)
        dec = self.decoder
        h = target.to(v.dtype)
        inter, inter_refs = [], []
        vr2 = torch.cat([valid_ratios, valid_ratios], -1)[:, None]
        for idx, layer in enumerate(dec.layers):
            ref_in = reference_points[:, :, None] * vr2
            query_pos = dec.reference_points_head(dec.proposal_pos_embed_rows(ref_in[:, :, 0, :], h.dtype))
            (h,) = layer(hidden_states=h, position_embeddings=query_pos, reference_points=ref_in.contiguous(),
                         spatial_shapes=spatial_shapes, level_start_index=lsi, vision_encoder_hidden_states=v,
                         vision_encoder_attention_mask=mask_flatten, text_encoder_hidden_states=t,
                         text_encoder_attention_mask=text_pad)
            if dec.bbox_embed is not None:
                reference_points = (dec.bbox_embed[idx](h) + inverse_sigmoid(reference_points)).sigmoid()
            inter.append(ops.layernorm(h, dec.layer_norm.weight, dec.layer_norm.bias, dec.layer_norm.eps))
            inter_refs.append(reference_points)
        return SimpleNamespace(init_reference_points=init_reference_points, intermediate_hidden_states=inter,
                               intermediate_reference_points=inter_refs, mask_features=mask_features,
                               encoder_last_hidden_state_vision=v, encoder_last_hidden_state_text=t,
                               enc_outputs_class=enc_class, enc_outputs_coord_logits=enc_coord, topk_proposals=topk_idx,
                               enc_topk_coords_logits=enc_topk_coords, enc_topk_class_logits=enc_topk_class,
                               spatial_shapes=spatial_shapes, level_start_index=lsi, valid_ratios=valid_ratios)


class B200GroundingDinoForObjectDetection(nn.Module):
    """Drop-in for `OVGroundingDinoForObjectDetection` at test time: same ctor config, same state-dict keys (shared
    bbox / mask heads appear once per decoder layer exactly as in the reference, gd.py:2617-2646), `forward` =
    `forward_test` -> object with `.logits [B,Q,max_text_len]`, `.pred_boxes [B,Q,4]`, `.pred_masks [B,Q,H/4,W/4]`
    in fp32 (gd.py:3193-3208)."""

    def __init__(self, config, backbone_model=None):
        super().__init__()
        self.config = config
        self.model = B200GroundingDinoModel(config, backbone_model)
        d, L = config.d_model, config.decoder_layers
        _class = H.GroundingDinoContrastiveEmbedding(config)
        _bbox = H.GroundingDinoMLPPredictionHead(d, d, 4, 3)
        _mask = H.GroundingDinoMLPPredictionHead(d, d, config.mask_dim, 3)
        self.mask_embed = nn.ModuleList([_mask for _ in range(L)])
        if not config.decoder_bbox_embed_share:
            raise NotImplementedError("per-layer bbox heads")
        self.bbox_embed = nn.ModuleList([_bbox for _ in range(L)])
        self.class_embed = nn.ModuleList([_class for _ in range(L)])
        self.model.decoder.bbox_embed = self.bbox_embed
        self.patch2query = H.GroundingDinoMLPPredictionHead(config.l_hidden_size, d, d, 3)

    @torch.no_grad()
    def forward_test(self, pixel_values, pixel_mask=None, text_query=None, text_query_masks=None, img_metas=None,
                     labels=None, all_levels=False, **unused):
        text = H.patch2query_mean(self.patch2query, text_query)
        out = self.model(pixel_values, pixel_mask=pixel_mask, text_query=text, text_query_masks=text_query_masks)
        mask_bool = text_query_masks.bool()
        n_levels = len(out.intermediate_hidden_states)
        res = []
        for level in (range(n_levels) if all_levels else [n_levels - 1]):
            ref = out.init_reference_points if level == 0 else out.intermediate_reference_points[level - 1]
            hs = out.intermediate_hidden_states[level]
            masks = H.forward_seg_heads(self.mask_embed[level], hs, out.mask_features,
                                        out_dtype=torch.float32 if hs.is_cuda and hs.dtype == torch.bfloat16 else None)
            logits = self.class_embed[level](hs, out.encoder_last_hidden_state_text, mask_bool)
            boxes = (self.bbox_embed[level](hs) + inverse_sigmoid(ref)).sigmoid()
            res.append((logits.to(torch.float32), boxes.to(torch.float32), masks.to(torch.float32)))
        logits, boxes, masks = res[-1]
        o = SimpleNamespace(logits=logits, pred_boxes=boxes, pred_masks=masks, model_outputs=out)
        if all_levels:
            o.aux = res
        return o

    def forward(self, pixel_values, pixel_mask=None, labels=None, **kw):
        if self.training or labels is not None:
            raise NotImplementedError("training path (contrastive DN + losses, gd.py:2659-3122) is out of scope")
        return self.forward_test(pixel_values, pixel_mask=pixel_mask, **kw)
