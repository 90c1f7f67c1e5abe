"""H100-native UniPose deformable layers (SURVEY.md 8f rank 4): drop-ins for
`MSDeformAttn` (visionllmv2/model/unipose/ops/modules/ms_deform_attn.py:33-158),
`DeformableTransformerEncoderLayer` and `DeformableTransformerDecoderLayer`
(visionllmv2/model/unipose/modeling_unipose.py:3132-3186, 3188-3323) -- the consumers of the MSDA operator in the
pose-estimation decoder.  Same constructor arguments, parameter names (`self_attn.{sampling_offsets,attention_weights,
value_proj,output_proj}`, `norm1/2/3`, `linear1/2`, `ca_text`, `catext_norm`, nn.MultiheadAttention's
`in_proj_weight/in_proj_bias/out_proj`) and call signatures (sequence-first `[nq, bs, d]` tensors in the decoder layer,
`True = padding` masks), on the kernels of the Grounding-DINO layers (visionllm_b200/gdino.py): packed
offsets|weights GEMM, MSDA kernel, fused attention, GEMM epilogues (+bias, ReLU/GELU, +residual), LayerNorm kernel.
Forward only; dropouts are identities at eval like in the reference.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .gdino import GroundingDinoMultiscaleDeformableAttention, _LN, _MHA


class MSDeformAttn(GroundingDinoMultiscaleDeformableAttention):
    """ms_deform_attn.py:33-158.  `input_padding_mask`: True = padding (the GDINO module takes True = valid)."""

    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4, use_4D_normalizer=False):
        super().__init__(SimpleNamespace(d_model=d_model, num_feature_levels=n_levels), num_heads=n_heads,
                         n_points=n_points)
        if use_4D_normalizer:
            raise NotImplementedError("use_4D_normalizer (never set by the UniPose builders, modeling_unipose.py:3144,3200)")
        self.use_4D_normalizer = use_4D_normalizer

    @torch.no_grad()
    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None):
        valid = None if input_padding_mask is None else ~input_padding_mask
        out, _ = super().forward(hidden_states=query, attention_mask=valid, encoder_hidden_states=input_flatten,
                                 encoder_attention_mask=valid, position_embeddings=None,
                                 reference_points=reference_points, spatial_shapes=input_spatial_shapes,
                                 level_start_index=input_level_start_index)
        return out


def _activation(name):
    if name not in ("relu", "gelu"):
        raise NotImplementedError(f"activation={name} (the UniPose configs use relu)")
    return name


class DeformableTransformerEncoderLayer(nn.Module):
    """modeling_unipose.py:3132-3186."""

    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4,
                 add_channel_attention=False, use_deformable_box_attn=False, box_attn_type="roi_align"):
        super().__init__()
        if add_channel_attention:
            raise NotImplementedError("add_channel_attention (DyReLU branch, off in the UniPose configs)")
        self.self_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.norm1 = _LN(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.act = _activation(activation)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.norm2 = _LN(d_model)
        self.add_channel_attention = False

    @staticmethod
    def with_pos_embed(tensor, pos):
        return tensor if pos is None else tensor + pos

    @torch.no_grad()
    def forward_ffn(self, src):
        h = ops.linear(src, self.linear1.weight, bias=self.linear1.bias, act=self.act)
        return self.norm2(ops.linear(h, self.linear2.weight, bias=self.linear2.bias, residual=src))

    @torch.no_grad()
    def forward(self, src, pos, reference_points, spatial_shapes, level_start_index, key_padding_mask=None):
        src2 = self.self_attn(self.with_pos_embed(src, pos), reference_points, src, spatial_shapes, level_start_index,
                              key_padding_mask)
        return self.forward_ffn(self.norm1(src + src2))


_ATTEND_CACHE = {}          # single entry: the last self-attention mask in kernel format (see _attend_mask)
_CONST_CACHE = {}           # small constant index tensors per (values, device): built once, so a forward issues no H2D copy


def _const_long(values, device, shape=None):
    key = (tuple(values) if shape is None else tuple(tuple(v) for v in values), str(device))
    t = _CONST_CACHE.get(key)
    if t is None:
        t = _CONST_CACHE[key] = torch.tensor(values, dtype=torch.long, device=device)
    return t


class DeformableTransformerDecoderLayer(nn.Module):
    """modeling_unipose.py:3188-3323: self-attention, optional text cross-attention, deformable cross-attention, FFN;
    tensors are sequence-first ([nq, bs, d]) like the reference's nn.MultiheadAttention calls."""

    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4,
                 use_text_feat_guide=False, use_text_cross_attention=False, ffn_extra_layernorm=False):
        super().__init__()
        assert not use_text_feat_guide
        if ffn_extra_layernorm:
            raise NotImplementedError("ffn_extra_layernorm not implemented")         # the reference raises too (:3222)
        self.cross_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.norm1 = _LN(d_model)
        if use_text_cross_attention:
            self.ca_text = _MHA(d_model, n_heads, dropout=dropout)
            self.catext_norm = _LN(d_model)
        self.self_attn = _MHA(d_model, n_heads, dropout=dropout)
        self.norm2 = _LN(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.act = _activation(activation)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.norm3 = _LN(d_model)
        self.norm_ext = None
        self.key_aware_proj = None
        self.use_text_feat_guide = use_text_feat_guide
        self.use_text_cross_attention = use_text_cross_attention
        self.n_heads = n_heads

    def rm_self_attn_modules(self):
        self.self_attn = None
        self.norm2 = None

    @staticmethod
    def with_pos_embed(tensor, pos):
        return tensor if pos is None else tensor + pos

    @torch.no_grad()
    def forward_ffn(self, tgt):
        h = ops.linear(tgt, self.linear1.weight, bias=self.linear1.bias, act=self.act)
        return self.norm3(ops.linear(h, self.linear2.weight, bias=self.linear2.bias, residual=tgt))

    def _attend_mask(self, self_attn_mask, bs, nq):
        """nn.MultiheadAttention attn_mask ([nq, nq] or [bs*heads, nq, nq], bool True = blocked) -> the kernel's
        [bs*heads, nq, nq] 'may attend' mask."""
        if self_attn_mask is None:
            return None
        if self_attn_mask.dtype != torch.bool:
            raise NotImplementedError("float attn_mask")
        # every keypoint layer receives the SAME mask tensor (tgt_mask2, 50 x 69 queries: 8 x 3450 x 3450 bytes per image):
        # invert / expand / convert it once per forward, not once per layer.  The cache entry keeps the source tensor alive, so
        # an `is` + version match cannot be a recycled allocation.
        c = _ATTEND_CACHE
        if c.get("src") is self_attn_mask and c.get("key") == (self_attn_mask._version, bs * self.n_heads, nq):
            return c["mask"]
        m = ~self_attn_mask
        if m.dim() == 2:
            m = m[None].expand(bs * self.n_heads, nq, nq)
        m = m.contiguous().view(torch.uint8)                       # the kernel's mask format: the bool bytes (0 / 1) reinterpreted
        if m.is_cuda and nq >= 256 and self.self_attn is not None and (self.self_attn.embed_dim // self.n_heads) in (32, 64, 128):
            # the keypoint layers' 50 x (1 + num_body_points) group mask is > 95 % blocked: list the live 64 x 64 tiles once and
            # let the attention kernel walk only those (bit-identical to the dense walk)
            m = ops.attention_mask_tiles(m)
        c.update(src=self_attn_mask, key=(self_attn_mask._version, bs * self.n_heads, nq), mask=m)
        return m

    @torch.no_grad()
    def forward(self, tgt, tgt_query_pos=None, tgt_query_sine_embed=None, tgt_key_padding_mask=None,
                tgt_reference_points=None, memory_text=None, text_attention_mask=None, memory=None,
                memory_key_padding_mask=None, memory_level_start_index=None, memory_spatial_shapes=None,
                memory_pos=None, self_attn_mask=None, cross_attn_mask=None):
        assert cross_attn_mask is None
        x = tgt.transpose(0, 1).contiguous()                                   # [bs, nq, d]
        pos = None if tgt_query_pos is None else tgt_query_pos.transpose(0, 1)
        bs, nq, _ = x.shape
        if self.self_attn is not None:
            qk = self.with_pos_embed(x, pos)
            x = self.norm2(self.self_attn.run(qk, qk, x, attn_mask=self._attend_mask(self_attn_mask, bs, nq), residual=x))
        if self.use_text_cross_attention:
            x = self.catext_norm(self.ca_text.run(self.with_pos_embed(x, pos), memory_text, memory_text,
                                                  key_mask=None if text_attention_mask is None else ~text_attention_mask,
                                                  residual=x))
        attn = self.cross_attn(self.with_pos_embed(x, pos), tgt_reference_points.transpose(0, 1).contiguous(),
                               memory.transpose(0, 1), memory_spatial_shapes, memory_level_start_index,
                               memory_key_padding_mask)
        x = self.forward_ffn(self.norm1(x + attn))
        return x.transpose(0, 1)


# ---------------------------------------------------------------------------------------------------------------------
# The two-stage keypoint decoder (modeling_unipose.py:2869-3130) and its heads
# ---------------------------------------------------------------------------------------------------------------------
import copy   # noqa: E402
import math   # noqa: E402

from .gdino_heads import GroundingDinoMLPPredictionHead as MLP   # noqa: E402  same `layers.N` parameters as utils/model_utils.py:147-160


def inverse_sigmoid(x, eps=1e-3):
    """utils/misc.py:667-671 (the variant modeling_unipose.py imports, eps = 1e-3)."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


def gen_sineembed_for_position(pos_tensor):
    """utils/model_utils.py:178-204: 128 sine features per coordinate, order (y, x[, w, h]), fp32 arithmetic."""
    scale = 2 * math.pi
    dim_t = torch.arange(128, dtype=torch.float32, device=pos_tensor.device)
    dim_t = 10000 ** (2 * (dim_t // 2) / 128)

    def emb(c):
        p = (pos_tensor[:, :, c] * scale)[:, :, None] / dim_t
        return torch.stack((p[:, :, 0::2].sin(), p[:, :, 1::2].cos()), dim=3).flatten(2)

    if pos_tensor.size(-1) == 2:
        return torch.cat((emb(1), emb(0)), dim=2)
    if pos_tensor.size(-1) == 4:
        return torch.cat((emb(1), emb(0), emb(2), emb(3)), dim=2)
    raise ValueError("Unknown pos_tensor shape(-1):{}".format(pos_tensor.size(-1)))


class ContrastiveAssign(nn.Module):
    """modeling_unipose.py:947-992: logits = x @ encoded_text^T, -inf on padded text tokens (already max_text_len wide)."""

    def __init__(self, project=False, cal_bias=None, max_text_len=256):
        super().__init__()
        if cal_bias is not None:
            raise NotImplementedError("cal_bias (the reference raises too, :979)")
        self.project, self.cal_bias, self.max_text_len = project, cal_bias, max_text_len

    @torch.no_grad()
    def forward(self, x, text_dict):
        y, mask = text_dict["encoded_text"], text_dict["text_token_mask"]
        B, Q, _ = x.shape
        T = y.shape[1]
        buf = torch.empty((B, Q, (T + 7) // 8 * 8), dtype=x.dtype, device=x.device)     # 16-byte output row pitch
        for b in range(B):
            ops.linear(x[b].contiguous(), y[b].to(x.dtype).contiguous(), out=buf[b, :, :T])
        res = buf[..., :T].masked_fill(~mask[:, None, :], float("-inf"))
        return res.float()                                     # `new_res` is a default-dtype (fp32) buffer (:988-990)


def _get_clones(module, N, layer_share=False):
    return nn.ModuleList([module for _ in range(N)] if layer_share else [copy.deepcopy(module) for _ in range(N)])


class TransformerDecoder(nn.Module):
    """modeling_unipose.py:2869-3130, inference path: `num_box_decoder_layers` box layers over the proposal queries, then
    the 50 best boxes (top-k of the max class logit, indices exact) are expanded into (1 box + num_body_points keypoint)
    queries each and refined by the remaining layers.  Same constructor arguments, parameter names (`layers.N`, `norm`,
    `ref_point_head.layers.N`, `hw`, `hw_append`) and late-bound heads (`bbox_embed`, `class_embed`, `pose_embed`,
    `pose_hw_embed` are assigned by the owner model, :233-239); sequence-first tensors; returns
    `[intermediate (bs-first), reference points (bs-first)]`.  Denoising queries exist only in training (:2985)."""

    def __init__(self, decoder_layer, num_layers, norm=None, return_intermediate=False, d_model=256, query_dim=4,
                 modulate_hw_attn=False, num_feature_levels=1, deformable_decoder=False, decoder_query_perturber=None,
                 dec_layer_number=None, rm_dec_query_scale=False, dec_layer_share=False, dec_layer_dropout_prob=None,
                 use_detached_boxes_dec_out=False, num_box_decoder_layers=2, num_body_points=68):
        super().__init__()
        self.layers = _get_clones(decoder_layer, num_layers, layer_share=dec_layer_share) if num_layers > 0 else []
        self.num_layers, self.norm = num_layers, norm
        assert return_intermediate, "support return_intermediate only"
        assert query_dim in (2, 4)
        self.return_intermediate, self.query_dim = return_intermediate, query_dim
        self.num_feature_levels, self.use_detached_boxes_dec_out = num_feature_levels, use_detached_boxes_dec_out
        self.ref_point_head = MLP(query_dim // 2 * d_model, d_model, d_model, 2)
        self.query_pos_sine_scale = None if deformable_decoder else MLP(d_model, d_model, d_model, 2)
        if not rm_dec_query_scale:
            raise NotImplementedError("query_scale (the reference raises too, :2908)")
        self.query_scale = None
        self.bbox_embed = self.class_embed = self.pose_embed = self.pose_hw_embed = None
        self.d_model, self.modulate_hw_attn, self.deformable_decoder = d_model, modulate_hw_attn, deformable_decoder
        self.ref_anchor_head = MLP(d_model, d_model, 2, 2) if (not deformable_decoder and modulate_hw_attn) else None
        if decoder_query_perturber is not None or dec_layer_number is not None or dec_layer_dropout_prob is not None:
            raise NotImplementedError("training-time query perturbation / per-layer query counts / layer dropout")
        self.decoder_query_perturber = self.dec_layer_number = self.dec_layer_dropout_prob = None
        self.rm_detach, self.box_pred_damping = None, None
        self.num_body_points = num_body_points
        self.hw = nn.Embedding(17, 2)
        self.num_box_decoder_layers = num_box_decoder_layers
        self.kpt_index = [x for x in range(50 * (num_body_points + 1)) if x % (num_body_points + 1) != 0]
        self.hw_append = nn.Embedding(num_body_points - 17, 2)

    @torch.no_grad()
    def forward(self, tgt, memory, tgt_mask=None, tgt_mask2=None, memory_mask=None, tgt_key_padding_mask=None,
                memory_key_padding_mask=None, pos=None, refpoints_unsigmoid=None, level_start_index=None,
                spatial_shapes=None, valid_ratios=None, memory_text=None, text_attention_mask=None, text_dict=None,
                dn_meta=None, targets=None, kpt_embed=None):
        if self.training:
            raise NotImplementedError("training (denoising queries) is outside the forward hot path")
        nbp, d = self.num_body_points, self.d_model
        output = tgt
        reference_points = refpoints_unsigmoid.sigmoid()
        intermediate, ref_points = [], [reference_points]
        kpt_index = _const_long(self.kpt_index, tgt.device)
        new_reference_points = None
        for layer_id, layer in enumerate(self.layers):
            if reference_points.shape[-1] == 4:
                rp_in = reference_points[:, :, None] * torch.cat([valid_ratios, valid_ratios], -1)[None, :]
            else:
                rp_in = reference_points[:, :, None] * valid_ratios[None, :]
            query_sine_embed = gen_sineembed_for_position(rp_in[:, :, 0, :]).to(tgt.dtype)
            query_pos = self.ref_point_head(query_sine_embed)
            output = layer(tgt=output, tgt_query_pos=query_pos, tgt_query_sine_embed=query_sine_embed,
                           tgt_key_padding_mask=tgt_key_padding_mask, tgt_reference_points=rp_in,
                           memory_text=memory_text, text_attention_mask=text_attention_mask, memory=memory,
                           memory_key_padding_mask=memory_key_padding_mask, memory_level_start_index=level_start_index,
                           memory_spatial_shapes=spatial_shapes, memory_pos=pos, self_attn_mask=tgt_mask,
                           cross_attn_mask=memory_mask).contiguous()
            intermediate.append(self.norm(output))
            if layer_id < self.num_box_decoder_layers:                          # box refinement (:3047-3051)
                new_reference_points = (self.bbox_embed[layer_id](output) + inverse_sigmoid(reference_points)).sigmoid()
            if layer_id == self.num_box_decoder_layers - 1:                     # pick 50 boxes, spawn keypoint queries
                cls = self.class_embed[layer_id](output.transpose(0, 1), text_dict).transpose(0, 1)   # [nq, bs, k]
                topk = torch.topk(cls.max(-1)[0], 50, dim=0)[1]                                       # [50, bs]
                if getattr(self, "forced_topk", None) is not None:   # compare runs of different precision on ONE selection
                    topk = self.forced_topk.to(topk.device)
                self.topk_proposals = topk                      # kept for inspection (the reference does not return it)
                box_ref = torch.gather(new_reference_points, 0, topk.unsqueeze(-1).repeat(1, 1, 4))
                box_out = torch.gather(output, 0, topk.unsqueeze(-1).repeat(1, 1, d))
                kpt_out = kpt_embed.transpose(0, 1)[None].repeat(box_out.shape[0], 1, 1, 1).to(output.dtype)   # [50, nkpt, bs, d]
                delta_xy = self.pose_embed[-1](kpt_out)[..., :2]
                kpt_xy = (inverse_sigmoid(box_ref[..., :2][:, None]) + delta_xy).sigmoid()
                nq2, _, bs, _ = kpt_xy.shape
                hw = torch.cat((self.hw.weight, self.hw_append.weight), dim=0)
                kpt_wh = hw.unsqueeze(0).unsqueeze(-2).repeat(nq2, 1, bs, 1).sigmoid() * box_ref[..., 2:][:, None]
                kpt_ref = torch.cat((kpt_xy, kpt_wh.to(kpt_xy.dtype)), dim=-1)
                new_reference_points = torch.cat((box_ref.unsqueeze(1), kpt_ref), dim=1).flatten(0, 1)
                output = torch.cat((box_out.unsqueeze(1), kpt_out), dim=1).flatten(0, 1)
                tgt_mask = tgt_mask2
            if layer_id >= self.num_box_decoder_layers:                         # box + keypoint refinement (:3103-3131)
                before = inverse_sigmoid(reference_points)
                j = layer_id - self.num_box_decoder_layers
                box_new = (self.bbox_embed[layer_id](output[0::(nbp + 1)].contiguous()) + before[0::(nbp + 1)]).sigmoid()
                out_kpt = output.index_select(0, kpt_index)
                unsig = before.index_select(0, kpt_index).clone()
                unsig[..., :2] += self.pose_embed[j](out_kpt)[..., :2]
                unsig[..., 2:] += self.pose_hw_embed[j](out_kpt)
                bs = box_new.shape[1]
                new_reference_points = torch.cat((box_new.unsqueeze(1), unsig.sigmoid().view(-1, nbp, bs, 4)),
                                                 dim=1).flatten(0, 1)
            reference_points = new_reference_points.detach()
            ref_points.append(reference_points if self.use_detached_boxes_dec_out else new_reference_points)
        return [[o.transpose(0, 1) for o in intermediate], [r.transpose(0, 1) for r in ref_points]]


def prepare_for_mask(kpt_mask, nheads, num_body_points, num_group=50):
    """UniPose.prepare_for_mask (modeling_unipose.py:887-917), the inference-time self-attention mask of the expanded
    (box + keypoint) queries, vectorised and on kpt_mask's device (the reference hard-codes 'cuda' and loops over
    50 * num_body_points rows).  kpt_mask [bs, 1 + num_body_points], 1 = the box slot / a real keypoint class.  Returns
    attn_mask2 [bs * nheads, T, T] bool, True = blocked, T = num_group * (1 + num_body_points).  Bug-compatible: the
    first pass groups rows by num_body_points (not 1 + num_body_points), so outside the diagonal blocks the pattern is
    the reference's, stripe for stripe."""
    bs, length = kpt_mask.shape
    dev = kpt_mask.device
    T = num_group * (1 + num_body_points)
    gb = num_body_points
    rows = torch.arange(T, device=dev)
    cols = torch.arange(T, device=dev)
    sj = (rows // gb) * gb
    ej = sj + gb
    touched = rows < num_group * gb
    left = (cols[None, :] < sj[:, None]) & (sj[:, None] > 0)
    right = (cols[None, :] >= ej[:, None]) & (ej[:, None] < num_group * gb)
    base = (left | right) & touched[:, None]                                    # [T, T]
    m = base[None].repeat(bs, 1, 1)
    equal = kpt_mask[:, :, None] == kpt_mask[:, None, :]                        # [bs, length, length]
    for idx in range(num_group):                                                # 50 diagonal blocks
        s0 = idx * length
        m[:, s0:s0 + length, s0:s0 + length] = ~equal
    return m[:, None].repeat(1, nheads, 1, 1).flatten(0, 1)


# ---------------------------------------------------------------------------------------------------------------------
# The UniPose transformer: text-fused deformable encoder, two-stage query selection, keypoint decoder
# (modeling_unipose.py:1943-2204 fusion / text layers, 2206-2700 DeformableTransformer, 2701-2868 TransformerEncoder)
# ---------------------------------------------------------------------------------------------------------------------
from . import gdino_heads as _H   # noqa: E402
from . import msda as _msda   # noqa: E402
from .gdino import get_sine_pos_embed   # noqa: E402


class BiMultiHeadAttention(nn.Module):
    """modeling_unipose.py:1943-2082 (parameter names v_proj / l_proj / values_v_proj / values_l_proj / out_v_proj /
    out_l_proj).  Both directions share S = (v_proj(v) * scale) l_proj(l)^T: softmax over the text keys updates the image
    tokens, softmax over the image keys of S^T the text tokens; the reference's global `S - S.max()` and +-50000 clamps do not
    change either softmax.  Masks: True = padding.  Two wgmma attention calls (head_dim = embed_dim / heads, 256 for the
    released config) on packed projection GEMMs."""

    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, cfg=None):
        super().__init__()
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        assert self.head_dim * num_heads == embed_dim
        self.v_dim, self.l_dim, self.scale, self.dropout = v_dim, l_dim, self.head_dim ** (-0.5), dropout
        self.v_proj, self.l_proj = nn.Linear(v_dim, embed_dim), nn.Linear(l_dim, embed_dim)
        self.values_v_proj, self.values_l_proj = nn.Linear(v_dim, embed_dim), nn.Linear(l_dim, embed_dim)
        self.out_v_proj, self.out_l_proj = nn.Linear(embed_dim, v_dim), nn.Linear(embed_dim, l_dim)
        self.stable_softmax_2d = self.clamp_min_for_underflow = self.clamp_max_for_overflow = True

    @torch.no_grad()
    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None, v_epilogue=None, l_epilogue=None):   # noqa: E741
        E, H, D = self.embed_dim, self.num_heads, self.head_dim
        wv = torch.cat([self.v_proj.weight, self.values_v_proj.weight], 0)
        bv = torch.cat([self.v_proj.bias, self.values_v_proj.bias], 0)
        wl = torch.cat([self.l_proj.weight, self.values_l_proj.weight], 0)
        bl = torch.cat([self.l_proj.bias, self.values_l_proj.bias], 0)
        pv = ops.linear(v, wv, bias=bv)                           # [B, S, 2E]: query side | values
        pl = ops.linear(l, wl, bias=bl)                           # [B, T, 2E]: key side | values
        vq, vval = pv[..., :E].unflatten(-1, (H, D)), pv[..., E:].unflatten(-1, (H, D))
        lk, lval = pl[..., :E].unflatten(-1, (H, D)), pl[..., E:].unflatten(-1, (H, D))
        km_l = None if attention_mask_l is None else ~attention_mask_l
        km_v = None if attention_mask_v is None else ~attention_mask_v
        v_ctx = ops.attention(vq, lk, lval, scale=self.scale, key_mask=km_l)      # image queries over text keys
        l_ctx = ops.attention(lk, vq, vval, scale=self.scale, key_mask=km_v)      # text queries over image keys
        dv = ops.linear(v_ctx, self.out_v_proj.weight, bias=self.out_v_proj.bias, **(v_epilogue or {}))
        dl = ops.linear(l_ctx, self.out_l_proj.weight, bias=self.out_l_proj.bias, **(l_epilogue or {}))
        return dv, dl


class BiAttentionBlock(nn.Module):
    """modeling_unipose.py:2169-2203: pre-LayerNorm, bi-attention, LayerScale (gam_v / gam_l) + residual ON THE NORMALISED
    features; LayerScale and residual ride in the output projections' GEMM epilogues."""

    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, drop_path=.0, init_values=1e-4, cfg=None):
        super().__init__()
        self.layer_norm_v, self.layer_norm_l = _LN(v_dim), _LN(l_dim)
        self.attn = BiMultiHeadAttention(v_dim=v_dim, l_dim=l_dim, embed_dim=embed_dim, num_heads=num_heads, dropout=dropout)
        self.drop_path = nn.Identity()
        self.gam_v = nn.Parameter(init_values * torch.ones((v_dim)), requires_grad=True)
        self.gam_l = nn.Parameter(init_values * torch.ones((l_dim)), requires_grad=True)

    @torch.no_grad()
    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None):   # noqa: E741
        v, l = self.layer_norm_v(v), self.layer_norm_l(l)   # noqa: E741
        return self.attn(v, l, attention_mask_v=attention_mask_v, attention_mask_l=attention_mask_l,
                         v_epilogue=dict(colscale=self.gam_v, residual=v), l_epilogue=dict(colscale=self.gam_l, residual=l))


class TransformerEncoderLayer(nn.Module):
    """modeling_unipose.py:2122-2166, the text enhancer: post-norm MHA + FFN on sequence-first [n_text, bs, d] tensors.
    `src_mask` [bs, nq, nk] bool (True = blocked) is expanded like the reference does -- `repeat(nhead, 1, 1)`, batch-minor,
    while nn.MultiheadAttention indexes batch-major: (batch b, head h) gets the mask of batch (b * nhead + h) % bs; identical
    for bs == 1, reproduced exactly for bs > 1.  `src_key_padding_mask` is ignored like in the reference (:2157)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False):
        super().__init__()
        assert not normalize_before
        self.self_attn = _MHA(d_model, nhead, dropout=dropout)
        self.linear1, self.linear2 = nn.Linear(d_model, dim_feedforward), nn.Linear(dim_feedforward, d_model)
        self.norm1, self.norm2 = _LN(d_model), _LN(d_model)
        self.act = _activation(activation)
        self.normalize_before, self.nhead = normalize_before, nhead

    @torch.no_grad()
    def forward(self, src, src_mask=None, src_key_padding_mask=None, pos=None):
        x = src.transpose(0, 1).contiguous()                                  # [bs, n, d]
        full = None
        if src_mask is not None:
            am = src_mask
            if am.dim() == 3 and am.shape[0] == x.shape[0]:
                am = am.repeat(self.nhead, 1, 1)
            elif am.dim() == 2:
                am = am[None].expand(x.shape[0] * self.nhead, -1, -1)
            full = ~am
        qk = x if pos is None else x + pos.transpose(0, 1).to(x.dtype)
        x = self.norm1(self.self_attn.run(qk, qk, x, attn_mask=full, residual=x))
        h = ops.linear(x, self.linear1.weight, bias=self.linear1.bias, act=self.act)
        x = self.norm2(ops.linear(h, self.linear2.weight, bias=self.linear2.bias, residual=x))
        return x.transpose(0, 1)


class TransformerEncoder(nn.Module):
    """modeling_unipose.py:2701-2866: per layer -- fusion (BiAttentionBlock), text enhancer, deformable layer."""

    def __init__(self, encoder_layer, num_layers, d_model=256, num_queries=300, enc_layer_share=False, text_enhance_layer=None,
                 feature_fusion_layer=None, use_checkpoint=False, use_transformer_ckpt=False):
        super().__init__()
        self.layers, self.text_layers, self.fusion_layers = [], [], []
        if num_layers > 0:
            self.layers = _get_clones(encoder_layer, num_layers, layer_share=enc_layer_share)
            if text_enhance_layer is not None:
                self.text_layers = _get_clones(text_enhance_layer, num_layers, layer_share=enc_layer_share)
            if feature_fusion_layer is not None:
                self.fusion_layers = _get_clones(feature_fusion_layer, num_layers, layer_share=enc_layer_share)
        self.query_scale, self.num_queries, self.num_layers, self.d_model = None, num_queries, num_layers, d_model

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        refs = []
        for lvl, (H_, W_) in enumerate(_msda.host_shape_list(spatial_shapes)):
            ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_, device=device),
                                          torch.linspace(0.5, W_ - 0.5, W_, device=device), indexing="ij")
            ref_y = ref_y.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * H_)
            ref_x = ref_x.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * W_)
            refs.append(torch.stack((ref_x, ref_y), -1))
        reference_points = torch.cat(refs, 1)
        return reference_points[:, :, None] * valid_ratios[:, None]

    @torch.no_grad()
    def forward(self, src, pos, spatial_shapes, level_start_index, valid_ratios, key_padding_mask, memory_text=None,
                text_attention_mask=None, pos_text=None, text_self_attention_masks=None, position_ids=None):
        output = src
        reference_points = None
        if self.num_layers > 0:
            reference_points = self.get_reference_points(spatial_shapes, valid_ratios.float(), device=src.device)
        if self.text_layers:
            bs, n_text, _ = memory_text.shape
            if pos_text is None and position_ids is None:
                pt = torch.arange(n_text, device=memory_text.device).float()[None, :, None].repeat(bs, 1, 1)
                pos_text = get_sine_pos_embed(pt, num_pos_feats=256, exchange_xy=False)
            if position_ids is not None:
                pos_text = get_sine_pos_embed(position_ids[..., None], num_pos_feats=256, exchange_xy=False)
        for layer_id, layer in enumerate(self.layers):
            if self.fusion_layers:
                output, memory_text = self.fusion_layers[layer_id](v=output, l=memory_text, attention_mask_v=key_padding_mask,
                                                                   attention_mask_l=text_attention_mask)
            if self.text_layers:
                memory_text = self.text_layers[layer_id](
                    src=memory_text.transpose(0, 1), src_mask=~text_self_attention_masks,
                    src_key_padding_mask=text_attention_mask,
                    pos=(pos_text.transpose(0, 1) if pos_text is not None else None)).transpose(0, 1)
            output = layer(src=output, pos=pos, reference_points=reference_points, spatial_shapes=spatial_shapes,
                           level_start_index=level_start_index, key_padding_mask=key_padding_mask)
        return output, memory_text


class DeformableTransformer(nn.Module):
    """modeling_unipose.py:2206-2700 for the configuration the UniPose builder produces (:4241-4330): deformable encoder
    and decoder, text enhancer + fusion layers, text cross-attention in the decoder, two-stage 'standard' query selection,
    learnable (`embed_init_tgt`) decoder queries.  Same constructor keywords and parameter names (`encoder.*`, `decoder.*`,
    `level_embed`, `tgt_embed`, `enc_output`, `enc_output_norm`; `enc_out_bbox_embed` / `enc_out_class_embed` and the
    decoder's heads are bound by the owner model, :233-257).  Unsupported switches raise."""

    def __init__(self, d_model=256, nhead=8, num_queries=300, num_encoder_layers=6, num_unicoder_layers=0, num_decoder_layers=6,
                 dim_feedforward=2048, dropout=0.0, activation="relu", normalize_before=False, return_intermediate_dec=False,
                 query_dim=4, num_patterns=0, modulate_hw_attn=False, deformable_encoder=False, deformable_decoder=False,
                 num_feature_levels=1, enc_n_points=4, dec_n_points=4, use_deformable_box_attn=False, box_attn_type='roi_align',
                 learnable_tgt_init=False, decoder_query_perturber=None, add_channel_attention=False, add_pos_value=False,
                 random_refpoints_xy=False, two_stage_type='standard', two_stage_pat_embed=0, two_stage_add_query_num=0,
                 two_stage_learn_wh=False, two_stage_keep_all_tokens=False, dec_layer_number=None, rm_enc_query_scale=True,
                 rm_dec_query_scale=True, rm_self_attn_layers=None, key_aware_type=None, layer_share_type=None, rm_detach=None,
                 decoder_sa_type='ca', module_seq=['sa', 'ca', 'ffn'], embed_init_tgt=False, use_detached_boxes_dec_out=False,
                 use_text_enhancer=False, use_fusion_layer=False, use_checkpoint=False, use_transformer_ckpt=False,
                 use_text_cross_attention=False, text_dropout=0.1, fusion_dropout=0.1, fusion_droppath=0.0,
                 binary_query_selection=False, ffn_extra_layernorm=False, num_box_decoder_layers=2, num_body_points=68):
        super().__init__()
        unsupported = dict(binary_query_selection=binary_query_selection, use_deformable_box_attn=use_deformable_box_attn,
                           add_channel_attention=add_channel_attention, two_stage_pat_embed=two_stage_pat_embed,
                           two_stage_add_query_num=two_stage_add_query_num, two_stage_learn_wh=two_stage_learn_wh,
                           two_stage_keep_all_tokens=two_stage_keep_all_tokens, rm_self_attn_layers=rm_self_attn_layers,
                           layer_share_type=layer_share_type, rm_detach=rm_detach, num_patterns=num_patterns,
                           normalize_before=normalize_before, ffn_extra_layernorm=ffn_extra_layernorm)
        bad = {k: v for k, v in unsupported.items() if v}
        if bad or not (deformable_encoder and deformable_decoder) or two_stage_type != 'standard' or query_dim != 4:
            raise NotImplementedError(f"DeformableTransformer: configuration outside the UniPose builder's ({bad})")
        assert learnable_tgt_init, "why not learnable_tgt_init"
        assert decoder_sa_type in ('sa', 'ca_label', 'ca_content')
        self.num_feature_levels, self.num_encoder_layers, self.num_decoder_layers = num_feature_levels, num_encoder_layers, num_decoder_layers
        self.num_queries, self.d_model, self.nhead, self.dec_layers = num_queries, d_model, nhead, num_decoder_layers
        self.two_stage_type, self.embed_init_tgt, self.decoder_sa_type = two_stage_type, embed_init_tgt, decoder_sa_type
        self.use_detached_boxes_dec_out = use_detached_boxes_dec_out
        encoder_layer = DeformableTransformerEncoderLayer(d_model, dim_feedforward, dropout, activation, num_feature_levels,
                                                          nhead, enc_n_points)
        text_layer = (TransformerEncoderLayer(d_model=d_model, nhead=nhead // 2, dim_feedforward=dim_feedforward // 2,
                                              dropout=text_dropout) if use_text_enhancer else None)
        fusion_layer = (BiAttentionBlock(v_dim=d_model, l_dim=d_model, embed_dim=dim_feedforward // 2, num_heads=nhead // 2,
                                         dropout=fusion_dropout, drop_path=fusion_droppath) if use_fusion_layer else None)
        self.encoder = TransformerEncoder(encoder_layer, num_encoder_layers, d_model=d_model, num_queries=num_queries,
                                          text_enhance_layer=text_layer, feature_fusion_layer=fusion_layer)
        decoder_layer = DeformableTransformerDecoderLayer(d_model, dim_feedforward, dropout, activation, num_feature_levels, nhead,
                                                          dec_n_points, use_text_cross_attention=use_text_cross_attention)
        self.decoder = TransformerDecoder(decoder_layer, num_decoder_layers, _LN(d_model), return_intermediate=return_intermediate_dec,
                                          d_model=d_model, query_dim=query_dim, modulate_hw_attn=modulate_hw_attn,
                                          num_feature_levels=num_feature_levels, deformable_decoder=deformable_decoder,
                                          rm_dec_query_scale=rm_dec_query_scale,
                                          use_detached_boxes_dec_out=use_detached_boxes_dec_out,
                                          num_box_decoder_layers=num_box_decoder_layers, num_body_points=num_body_points)
        self.level_embed = (nn.Parameter(torch.zeros(num_feature_levels, d_model))
                            if (num_feature_levels > 1 and num_encoder_layers > 0) else None)
        self.tgt_embed = nn.Embedding(num_queries, d_model) if embed_init_tgt else None
        self.enc_output, self.enc_output_norm = nn.Linear(d_model, d_model), _LN(d_model)
        self.two_stage_wh_embedding = None
        self.enc_out_class_embed = self.enc_out_bbox_embed = None

    @staticmethod
    def get_valid_ratio(mask):
        _, H, W = mask.shape
        valid_H, valid_W = torch.sum(~mask[:, :, 0], 1), torch.sum(~mask[:, 0, :], 1)
        return torch.stack([valid_W.float() / W, valid_H.float() / H], -1)

    @torch.no_grad()
    def forward(self, srcs, masks, refpoint_embed, pos_embeds, tgt, attn_mask=None, attn_mask2=None, text_dict=None,
                dn_meta=None, targets=None, kpt_embed=None):
        """srcs / pos_embeds: per-level [bs, c, h, w] maps, masks [bs, h, w] (True = padding); refpoint_embed / tgt: the
        denoising queries (training only: must be None).  Returns (hs, references, hs_enc, ref_enc, init_box_proposal)."""
        if refpoint_embed is not None or tgt is not None or self.training:
            raise NotImplementedError("denoising queries / training are outside the forward hot path")
        src_l, mask_l, pos_l, shapes = [], [], [], []
        for lvl, (src, mask, pos_embed) in enumerate(zip(srcs, masks, pos_embeds)):
            bs, c, h, w = src.shape
            shapes.append((h, w))
            src_l.append(src.flatten(2).transpose(1, 2))
            mask_l.append(mask.flatten(1))
            pe = pos_embed.flatten(2).transpose(1, 2)
            if self.num_feature_levels > 1 and self.level_embed is not None:
                pe = pe + self.level_embed[lvl].view(1, 1, -1)
            pos_l.append(pe)
        src_flatten, mask_flatten = torch.cat(src_l, 1).contiguous(), torch.cat(mask_l, 1)
        lvl_pos = torch.cat(pos_l, 1).contiguous()
        spatial_shapes = _const_long([tuple(int(v) for v in hw) for hw in shapes], src_flatten.device, shape=2)
        if getattr(spatial_shapes, "_b200_host", None) is None:
            _msda.attach_host_shapes(spatial_shapes, shapes)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
        valid_ratios = torch.stack([self.get_valid_ratio(m) for m in masks], 1)

        memory, memory_text = self.encoder(
            src_flatten, pos=lvl_pos, level_start_index=level_start_index, spatial_shapes=spatial_shapes,
            valid_ratios=valid_ratios, key_padding_mask=mask_flatten, memory_text=text_dict['encoded_text'],
            text_attention_mask=~text_dict['text_token_mask'], position_ids=text_dict['position_ids'],
            text_self_attention_masks=text_dict['text_self_attention_masks'])
        text_dict = dict(text_dict)
        text_dict['encoded_text'] = memory_text
        self.decoder_text = memory_text                      # the reference mutates the caller's text_dict (:2546); kept for the heads

        # two-stage 'standard' query selection (:2557-2606); top-k indices through torch.topk like the reference
        output_memory, output_proposals = _H.gen_encoder_output_proposals(self.enc_output, self.enc_output_norm, memory,
                                                                          mask_flatten, spatial_shapes)
        cls = self.enc_out_class_embed(output_memory, text_dict)
        topk_logits = cls.max(-1)[0]
        coord_unselected = self.enc_out_bbox_embed(output_memory).float() + output_proposals
        topk_proposals = torch.topk(topk_logits, self.num_queries, dim=1)[1]
        if getattr(self, "forced_topk", None) is not None:
            topk_proposals = self.forced_topk.to(topk_proposals.device)
        self.topk_proposals = topk_proposals
        refpoint_undetach = torch.gather(coord_unselected, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4))
        init_box_proposal = torch.gather(output_proposals, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4)).sigmoid()
        tgt_undetach = torch.gather(output_memory, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, self.d_model))
        bs = memory.shape[0]
        if self.embed_init_tgt:
            tgt_ = self.tgt_embed.weight[:, None, :].repeat(1, bs, 1).transpose(0, 1)
        else:
            tgt_ = tgt_undetach
        refpoint_embed, tgt = refpoint_undetach, tgt_.to(memory.dtype)

        hs, references = self.decoder(
            tgt=tgt.transpose(0, 1).contiguous(), memory=memory.transpose(0, 1), memory_key_padding_mask=mask_flatten,
            pos=lvl_pos.transpose(0, 1), refpoints_unsigmoid=refpoint_embed.transpose(0, 1),      # fp32, like the reference
            level_start_index=level_start_index, spatial_shapes=spatial_shapes, valid_ratios=valid_ratios,
            tgt_mask=attn_mask, tgt_mask2=attn_mask2, memory_text=text_dict['encoded_text'],
            text_attention_mask=~text_dict['text_token_mask'], text_dict=text_dict, dn_meta=dn_meta, targets=targets,
            kpt_embed=kpt_embed)
        hs_enc = tgt_undetach.unsqueeze(0)
        ref_enc = refpoint_undetach.sigmoid().unsqueeze(0)
        return hs, references, hs_enc, ref_enc, init_box_proposal


def generate_masks_with_text_query_masks(text_query_masks):
    """modeling_unipose.py:928-945: text_query_masks [bs, n] (1 = a real class token) -> (self_attention_mask [bs, n, n] bool:
    identity plus the all-pairs block of the first num_valid tokens; position_ids [bs, n]: 0..num_valid-1, then zeros).
    Vectorised (the reference loops over the batch with a device sync per sample)."""
    bs, n = text_query_masks.shape
    dev = text_query_masks.device
    nv = text_query_masks.sum(1).to(torch.long)                                   # [bs]
    ar = torch.arange(n, device=dev)
    inside = ar[None, :] < nv[:, None]                                           # [bs, n]
    mask = torch.eye(n, device=dev, dtype=torch.bool)[None].repeat(bs, 1, 1) | (inside[:, :, None] & inside[:, None, :])
    position_ids = torch.where(inside, ar[None, :].expand(bs, n), torch.zeros((), dtype=torch.long, device=dev))
    return mask, position_ids


# ---------------------------------------------------------------------------------------------------------------------
# The UniPose model behind its backbone (modeling_unipose.py:69-655, inference path)
# ---------------------------------------------------------------------------------------------------------------------
from .gdino_model import conv_rows as _conv_rows   # noqa: E402


class PositionEmbeddingSineHW(nn.Module):
    """modeling_unipose.py:1037-1078 (no parameters); takes the padding mask [bs, h, w] (True = padding), returns NCHW fp32."""

    def __init__(self, num_pos_feats=64, temperatureH=10000, temperatureW=10000, normalize=False, scale=None):
        super().__init__()
        if scale is not None and normalize is False:
            raise ValueError("normalize should be True if scale is passed")
        self.num_pos_feats, self.temperatureH, self.temperatureW, self.normalize = num_pos_feats, temperatureH, temperatureW, normalize
        self.scale = 2 * math.pi if scale is None else scale

    @torch.no_grad()
    def forward(self, mask):
        not_mask = ~mask
        y_embed, x_embed = not_mask.cumsum(1, dtype=torch.float32), not_mask.cumsum(2, dtype=torch.float32)
        if self.normalize:
            eps = 1e-6
            y_embed = y_embed / (y_embed[:, -1:, :] + eps) * self.scale
            x_embed = x_embed / (x_embed[:, :, -1:] + eps) * self.scale
        d = torch.arange(self.num_pos_feats, dtype=torch.float32, device=mask.device)
        pos_x = x_embed[:, :, :, None] / (self.temperatureW ** (2 * (d // 2) / self.num_pos_feats))
        pos_y = y_embed[:, :, :, None] / (self.temperatureH ** (2 * (d // 2) / self.num_pos_feats))
        pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
        pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
        return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)


def keypoint_xyzxyz_to_xyxyzz(keypoints):
    """utils/keypoint_ops.py:18-29: (x, y, z) triples -> all (x, y) pairs, then all z."""
    res = torch.zeros_like(keypoints)
    n = keypoints.shape[-1] // 3
    res[..., 0:2 * n:2] = keypoints[..., 0::3]
    res[..., 1:2 * n:2] = keypoints[..., 1::3]
    res[..., 2 * n:] = keypoints[..., 2::3]
    return res


class B200UniPose(nn.Module):
    """`UniPose` (modeling_unipose.py:69-655) behind its image backbone, inference path: [EMB]-state projections
    (`projection_llava`, `projection_kpt_llava`), `input_proj` (1x1 conv + GroupNorm per backbone level, 3x3 stride-2 conv +
    GroupNorm for the extra levels), the transformer above, and the box / class / keypoint heads with the reference's
    parameter names (shared heads repeated like its ModuleLists).  The backbone (`Joiner`: Swin + sine position embedding) is
    injected: `forward(features=[(map NCHW, mask)], poss=[NCHW], text_query=...)` takes what `self.backbone(samples)` returns.
    With `backbone=` (a `unipose_backbone.B200Joiner`, state-dict prefix `backbone.0.` like the reference's `self.backbone`)
    `forward_samples(tensors, mask, text_query)` is the reference's `forward(samples, None, text_query)` on the padded batch.
    """

    def __init__(self, hidden_dim=256, l_hidden_size=4096, backbone_channels=(192, 384, 768), num_feature_levels=4,
                 num_queries=900, num_body_points=68, num_box_decoder_layers=2, nheads=8, pe_temperatureH=20, pe_temperatureW=20,
                 transformer=None, backbone=None, **transformer_kwargs):
        super().__init__()
        if backbone is not None:
            self.backbone = backbone
        self.hidden_dim, self.num_feature_levels, self.num_queries, self.nheads = hidden_dim, num_feature_levels, num_queries, nheads
        self.num_body_points, self.num_box_decoder_layers = num_body_points, num_box_decoder_layers
        self.transformer = transformer if transformer is not None else DeformableTransformer(
            d_model=hidden_dim, nhead=nheads, num_queries=num_queries, num_feature_levels=num_feature_levels,
            num_box_decoder_layers=num_box_decoder_layers, num_body_points=num_body_points, **transformer_kwargs)
        self.position_embedding = PositionEmbeddingSineHW(hidden_dim // 2, pe_temperatureH, pe_temperatureW, normalize=True)
        self.projection_llava = MLP(l_hidden_size, hidden_dim, hidden_dim, 3)
        self.projection_kpt_llava = MLP(l_hidden_size, hidden_dim, hidden_dim, 3)
        proj, cin = [], None
        for cin in backbone_channels:
            proj.append(nn.Sequential(nn.Conv2d(cin, hidden_dim, kernel_size=1), nn.GroupNorm(32, hidden_dim)))
        for _ in range(num_feature_levels - len(backbone_channels)):
            proj.append(nn.Sequential(nn.Conv2d(cin, hidden_dim, kernel_size=3, stride=2, padding=1), nn.GroupNorm(32, hidden_dim)))
            cin = hidden_dim
        self.input_proj = nn.ModuleList(proj)
        n_dec = self.transformer.num_decoder_layers
        bbox, pose, pose_hw, cls = MLP(hidden_dim, hidden_dim, 4, 3), MLP(hidden_dim, hidden_dim, 2, 3), MLP(hidden_dim, hidden_dim, 2, 3), ContrastiveAssign()
        self.bbox_embed = nn.ModuleList([bbox for _ in range(n_dec)])                      # dec_pred_bbox_embed_share (:166)
        self.class_embed = nn.ModuleList([cls for _ in range(n_dec)])
        self.pose_embed = nn.ModuleList([pose for _ in range(n_dec - num_box_decoder_layers + 1)])
        self.pose_hw_embed = nn.ModuleList([pose_hw for _ in range(n_dec - num_box_decoder_layers)])
        d = self.transformer.decoder
        d.bbox_embed, d.class_embed, d.pose_embed, d.pose_hw_embed = self.bbox_embed, self.class_embed, self.pose_embed, self.pose_hw_embed
        self.transformer.enc_out_bbox_embed = copy.deepcopy(bbox)                          # two_stage_bbox_embed_share = False (:249)
        self.transformer.enc_out_class_embed = copy.deepcopy(cls)

    @torch.no_grad()
    def _proj(self, idx, x_nchw):
        """input_proj[idx] (Conv2d + GroupNorm(32)) on a NCHW map -> NCHW, through the GEMM + GroupNorm kernels."""
        conv, gn = self.input_proj[idx][0], self.input_proj[idx][1]
        rows, Ho, Wo = _conv_rows(x_nchw.permute(0, 2, 3, 1).contiguous(), conv)
        y = ops.groupnorm_nhwc(rows, gn.weight, gn.bias, gn.num_groups, gn.eps)
        return y.reshape(x_nchw.shape[0], Ho, Wo, -1).permute(0, 3, 1, 2)

    @torch.no_grad()
    def forward_samples(self, tensors, mask, text_query):
        """`UniPose.forward(samples, None, text_query)` (:330-655): tensors [bs, 3, H, W] = the zero-padded batch of
        `nested_tensor_from_tensor_list`, mask [bs, H, W] bool (True = padding)."""
        if not hasattr(self, "backbone"):
            raise RuntimeError("B200UniPose was built without a backbone: pass backbone=build_backbone(...) or call forward() "
                               "with the backbone's maps")
        features, poss = self.backbone(tensors, mask)                                      # :430
        return self.forward(features, poss, text_query, sample_mask=mask)

    @torch.no_grad()
    def forward(self, features, poss, text_query, sample_mask=None):
        """features: [(map [bs, c_l, h_l, w_l], mask [bs, h_l, w_l])] per backbone level; poss: their position embeddings;
        text_query: {'obj_querys' [bs, n_obj, n_emb, C], 'obj_query_masks' [bs, n_obj], 'kpt_querys', 'kpt_query_masks'};
        sample_mask [bs, H, W]: the padded batch's pixel mask (needed when extra feature levels are derived, :434-438)."""
        if self.training:
            raise NotImplementedError("training (denoising queries, criterion) is outside the forward hot path")
        dt = features[0][0].dtype
        bs = text_query['obj_querys'].shape[0]
        encoded_text = self.projection_llava(text_query['obj_querys']).mean(-2)
        kpt_embed = torch.zeros((bs, self.num_body_points, self.hidden_dim), dtype=dt, device=features[0][0].device)
        kpt_all = self.projection_kpt_llava(text_query['kpt_querys']).mean(-2)
        n_kpt = text_query['kpt_query_masks'].sum(1)
        keep = torch.arange(kpt_all.shape[1], device=kpt_all.device)[None, :] < n_kpt[:, None]        # first n_kpt rows per sample
        nk = min(kpt_all.shape[1], self.num_body_points)
        kpt_embed[:, :nk] = torch.where(keep[:, :nk, None], kpt_all[:, :nk].to(dt), kpt_embed[:, :nk])
        kpt_vis = text_query["kpt_query_masks"][:, :self.num_body_points]
        kpt_mask = torch.cat((torch.ones_like(kpt_vis)[..., 0].unsqueeze(-1), kpt_vis), dim=-1)
        sa, pid = generate_masks_with_text_query_masks(text_query['obj_query_masks'])
        text_dict = {'encoded_text': encoded_text, 'text_token_mask': text_query['obj_query_masks'].bool(), 'position_ids': pid,
                     'text_self_attention_masks': sa}
        srcs, masks, poss = [], [], list(poss)
        for lvl, (src, mask) in enumerate(features):
            srcs.append(self._proj(lvl, src))
            masks.append(mask)
        for lvl in range(len(srcs), self.num_feature_levels):
            src = self._proj(lvl, features[-1][0] if lvl == len(features) else srcs[-1])
            mask = F.interpolate(sample_mask[None].float(), size=src.shape[-2:]).to(torch.bool)[0]
            srcs.append(src)
            masks.append(mask)
            poss.append(self.position_embedding(mask).to(src.dtype))
        attn_mask2 = prepare_for_mask(kpt_mask, self.nheads, self.num_body_points)
        hs, reference, hs_enc, ref_enc, init_box = self.transformer(srcs, masks, None, poss, None, None, attn_mask2, text_dict,
                                                                    None, None, kpt_embed)
        text_dict = dict(text_dict)
        nbp, nb = self.num_body_points, self.num_box_decoder_layers
        coords, classes, keypoints = [], [], []
        kpt_index = _const_long([x for x in range(50 * (nbp + 1)) if x % (nbp + 1) != 0], hs[0].device)
        text_dict['encoded_text'] = self.transformer.decoder_text if hasattr(self.transformer, "decoder_text") else text_dict['encoded_text']
        for lid, (ref_sig, bbox_embed, cls_embed, layer_hs) in enumerate(zip(reference[:-1], self.bbox_embed, self.class_embed, hs)):
            if lid < nb:
                coords.append((bbox_embed(layer_hs) + inverse_sigmoid(ref_sig)).sigmoid().to(torch.float32))
                classes.append(cls_embed(layer_hs, text_dict).to(torch.float32))
                keypoints.append(layer_hs.new_zeros((bs, self.num_queries, nbp * 3)).to(torch.float32))
            else:
                hs_box, ref_box = layer_hs[:, 0::(nbp + 1), :].contiguous(), ref_sig[:, 0::(nbp + 1), :]
                coords.append((bbox_embed(hs_box) + inverse_sigmoid(ref_box)).sigmoid().to(torch.float32))
                classes.append(cls_embed(hs_box, text_dict).to(torch.float32))
                hs_kpt = layer_hs.index_select(1, kpt_index)
                ref_kpt = ref_sig.index_select(1, kpt_index)
                xy_unsig = self.pose_embed[lid - nb](hs_kpt) + inverse_sigmoid(ref_kpt[..., :2])
                xyv = torch.cat((xy_unsig, torch.ones_like(xy_unsig)[:, :, 0].unsqueeze(-1)), dim=-1).sigmoid()
                keypoints.append(keypoint_xyzxyz_to_xyxyzz(xyv.reshape((bs, 50, nbp, 3)).flatten(2, 3)).to(torch.float32))
        return SimpleNamespace(loss=None, loss_dict=None, pred_logits=classes[-1], pred_boxes=coords[-1], pred_keypoints=keypoints[-1],
                               aux=dict(classes=classes, coords=coords, keypoints=keypoints, hs_enc=hs_enc, ref_enc=ref_enc))


@torch.no_grad()
def post_process_pose(pred_logits, pred_boxes, pred_keypoints, target_sizes, num_classes=1, topk=100, num_body_points=17,
                      id_mapping=None, threshold=0.):
    """eval_pose.py:19-86, the caller right after the UniPose path: sigmoid -> top-k over (query, class) -> `//`, `%` -> labels
    through `id_mapping` (continuous -> dataset category id) -> boxes cxcywh -> xyxy scaled to the image -> the selected
    queries' keypoints (x, y of the first `num_body_points`, scaled; visibility 1) re-interleaved xyxy..zz -> xyzxyz ->
    score threshold.  target_sizes: [bs, 2] tensor or list of (h, w).  The id mapping is one table lookup instead of the
    reference's per-element `.item()` loop (same integers)."""
    if id_mapping is None:
        raise ValueError("id_mapping is required (the reference asserts it, eval_pose.py:42)")
    if target_sizes is not None and len(pred_logits) != len(target_sizes):
        raise ValueError("Make sure that you pass in as many target sizes as the batch dimension of the logits")
    logits = pred_logits[:, :, :num_classes]
    bs, K = logits.shape[0], logits.shape[2]
    prob = logits.sigmoid().view(bs, -1)
    scores, idx = torch.topk(prob, min(topk, prob.size(1)), dim=1)
    q_idx = torch.div(idx, K, rounding_mode="floor")
    labels = idx % K
    keys = sorted(id_mapping)
    table = torch.zeros(max(keys) + 1, dtype=labels.dtype, device=labels.device)
    table[torch.tensor(keys, device=labels.device)] = torch.tensor([id_mapping[k] for k in keys], dtype=labels.dtype,
                                                                    device=labels.device)
    labels = table[labels]
    if not torch.is_tensor(target_sizes):
        target_sizes = torch.stack([torch.as_tensor(t) for t in target_sizes])
    img_h, img_w = target_sizes.to(pred_boxes.device).unbind(1)
    boxes = torch.gather(_H.box_cxcywh_to_xyxy(pred_boxes), 1, q_idx.unsqueeze(-1).repeat(1, 1, 4))
    boxes = boxes * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]
    kp = torch.gather(pred_keypoints, 1, q_idx.unsqueeze(-1).repeat(1, 1, pred_keypoints.shape[-1]))
    z = kp[:, :, :num_body_points * 2] * torch.stack([img_w, img_h], dim=1).repeat(1, num_body_points)[:, None, :]
    out = torch.zeros((bs, z.shape[1], num_body_points * 3), dtype=z.dtype, device=z.device)
    out[..., 0::3], out[..., 1::3], out[..., 2::3] = z[..., 0::2], z[..., 1::2], 1.0
    res = []
    for s_, l_, b_, k_ in zip(scores, labels, boxes, out):
        keep = s_ > threshold
        res.append({"scores": s_[keep], "labels": l_[keep], "boxes": b_[keep], "keypoints": k_[keep]})
    return res

