"""H100-native Grounding-DINO deformable blocks (the region/mask decoder's hot layers).

Same class names, constructor arguments, parameter names and call signatures as
visionllmv2/model/grounding_dino/modeling_ov_grounding_dino_mask_dn.py:
  GroundingDinoMultiscaleDeformableAttention  :646-784   (sampling_offsets / attention_weights / value_proj /
                                                           output_proj -> MSDA gather)
  GroundingDinoDeformableLayer                :1104-1182 (encoder: MSDA + LN + FFN + LN)
  GroundingDinoDecoderLayer                   :1292-1407 (self-MHA, text cross-MHA, MSDA cross-attn, FFN)
  GroundingDinoTextEnhancerLayer              :793-857   (text self-MHA 4x64 + FFN)
  GroundingDinoBiMultiHeadAttention           :860-1006  (vision<->text bi-attention, 4 heads x 256)
  GroundingDinoFusionLayer                    :1039-1102 (LN, bi-attention, LayerScale residuals)
  GroundingDinoEncoderLayer                   :1216-1289 (fusion -> text enhancer -> deformable layer)
so reference state dicts load unchanged and the modules can be assigned over the reference classes
(INTEGRATION.md).  Projections run on the wgmma GEMM (offset and weight projections share one launch),
LayerNorm/residuals on the row kernels, attention on the fused attention kernel, the gather on
vllm_msda_forward_f32 -- never the grid_sample fallback the reference silently drops to (:777-779).
Forward / inference only.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import msda as msda_ext
from . import ops


class GroundingDinoMultiscaleDeformableAttention(nn.Module):
    def __init__(self, config, num_heads, n_points):
        super().__init__()
        if config.d_model % num_heads != 0:
            raise ValueError(f"embed_dim (d_model) must be divisible by num_heads, but got {config.d_model} "
                             f"and {num_heads}")
        self.im2col_step = 64
        self.d_model = config.d_model
        self.n_levels = config.num_feature_levels
        self.n_heads = num_heads
        self.n_points = n_points
        self.sampling_offsets = nn.Linear(config.d_model, num_heads * self.n_levels * n_points * 2)
        self.attention_weights = nn.Linear(config.d_model, num_heads * self.n_levels * n_points)
        self.value_proj = nn.Linear(config.d_model, config.d_model)
        self.output_proj = nn.Linear(config.d_model, config.d_model)
        self._packed = None
        self._reset_parameters()

    # the reference module always returns the attention weights (gd.py:784); an owner that never reads them (the H100 GDINO
    # stage) clears this so the fused gather kernel skips the [B, Lq, M, L, P] side output
    need_weights = True

    def _reset_parameters(self):
        # same init as the reference (:688-706)
        nn.init.constant_(self.sampling_offsets.weight.data, 0.0)
        thetas = torch.arange(self.n_heads, dtype=torch.float32) * (2.0 * math.pi / self.n_heads)
        grid = torch.stack([thetas.cos(), thetas.sin()], -1)
        grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(self.n_heads, 1, 1, 2).repeat(
            1, self.n_levels, self.n_points, 1)
        for i in range(self.n_points):
            grid[:, :, i, :] *= i + 1
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(grid.view(-1))
        nn.init.constant_(self.attention_weights.weight.data, 0.0)
        nn.init.constant_(self.attention_weights.bias.data, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight.data)
        nn.init.constant_(self.value_proj.bias.data, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight.data)
        nn.init.constant_(self.output_proj.bias.data, 0.0)

    def _packed_query_proj(self, dtype):
        ws = (self.sampling_offsets.weight, self.attention_weights.weight, self.sampling_offsets.bias,
              self.attention_weights.bias)
        key = tuple((w.data_ptr(), w._version) for w in ws) + (dtype,)
        if self._packed is None or self._packed[0] != key:
            w = torch.cat([ws[0].detach(), ws[1].detach()], 0).to(dtype).contiguous()
            b = torch.cat([ws[2].detach(), ws[3].detach()], 0).to(dtype).contiguous()
            self._packed = (key, w, b)
        return self._packed[1], self._packed[2]

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None, encoder_attention_mask=None,
                position_embeddings=None, reference_points=None, spatial_shapes=None, level_start_index=None,
                output_attentions=False, residual=None):
        """residual (extension): added in the output projection's epilogue, so the caller's `x + attn` before its LayerNorm
        costs no extra pass (fp32 accumulator + bias + residual, one rounding instead of the reference's two)."""
        if position_embeddings is not None:
            hidden_states = hidden_states + position_embeddings
        B, Lq, _ = hidden_states.shape
        _, S, _ = encoder_hidden_states.shape
        if sum(h * w for h, w in msda_ext.host_shape_list(spatial_shapes)) != S:      # host copy if attached: no sync
            raise ValueError("Make sure to align the spatial shapes with the sequence length of the encoder "
                             "hidden states")
        M, L, P, D = self.n_heads, self.n_levels, self.n_points, self.d_model // self.n_heads
        # padded pixels are zeroed in `value` before the op (gd.py:730-732): a row mask of the projection's epilogue
        value = ops.linear(encoder_hidden_states, self.value_proj.weight, bias=self.value_proj.bias,
                           row_keep=attention_mask)
        w, b = self._packed_query_proj(hidden_states.dtype)
        qp = ops.linear(hidden_states, w, bias=b)                    # offsets | weights in one GEMM
        n_off = M * L * P * 2
        if (reference_points.shape[-1] == 2 and Lq == S and value.dtype == torch.bfloat16 and P == 4
                and self.output_proj.weight.dtype == torch.bfloat16):
            # encoder self-attention: softmax / offset normalisation / reference add run inside the gather kernel
            fused = msda_ext.ms_deform_attn_forward_fused(value.view(B, S, M, D), spatial_shapes, level_start_index, qp,
                                                          reference_points, self.output_proj.weight.dtype,
                                                          want_weights=self.need_weights or output_attentions)
            if fused is not None:
                out, attention_weights = fused
                return ops.linear(out, self.output_proj.weight, bias=self.output_proj.bias, residual=residual), attention_weights
        sampling_offsets = qp[..., :n_off].reshape(B, Lq, M, L, P, 2)
        attention_weights = F.softmax(qp[..., n_off:].reshape(B, Lq, M, L * P), -1).view(B, Lq, M, L, P)
        if reference_points.shape[-1] == 2:
            normalizer = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
            loc = reference_points[:, :, None, :, None, :] + sampling_offsets / normalizer[None, None, None, :, None, :]
        elif reference_points.shape[-1] == 4:
            loc = (reference_points[:, :, None, :, None, :2]
                   + sampling_offsets / self.n_points * reference_points[:, :, None, :, None, 2:] * 0.5)
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but got {reference_points.shape[-1]}")
        # the reference upcasts value / weights to fp32 for its fp32-only kernel (:764-766); locations follow type
        # promotion.  With a bf16 value we read it in place (exact upcast inside the kernel) and write bf16 directly.
        if value.dtype == torch.bfloat16 and msda_ext.supports_bf16_value(D, L, P):
            out = msda_ext.ms_deform_attn_forward_bf16(value.view(B, S, M, D), spatial_shapes, level_start_index,
                                                       loc.float().contiguous(), attention_weights.float().contiguous(),
                                                       self.output_proj.weight.dtype)
        else:
            out = msda_ext.ms_deform_attn_forward(value.view(B, S, M, D).float().contiguous(), spatial_shapes,
                                                  level_start_index, loc.float().contiguous(),
                                                  attention_weights.float().contiguous(), self.im2col_step)
            out = out.to(self.output_proj.weight.dtype)
        out = ops.linear(out, self.output_proj.weight, bias=self.output_proj.bias, residual=residual)
        return out, attention_weights


def _act(config):
    a = getattr(config, "activation_function", "relu")
    if a not in ("relu", "gelu", "silu"):
        raise NotImplementedError(f"activation_function={a}")
    return a


class _LN(nn.LayerNorm):
    def forward(self, x):
        return ops.layernorm(x, self.weight, self.bias, self.eps)


class GroundingDinoDeformableLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embed_dim = config.d_model
        self.self_attn = GroundingDinoMultiscaleDeformableAttention(
            config, num_heads=config.encoder_attention_heads, n_points=config.encoder_n_points)
        self.self_attn_layer_norm = _LN(self.embed_dim)
        self.act = _act(config)
        self.fc1 = nn.Linear(self.embed_dim, config.encoder_ffn_dim)
        self.fc2 = nn.Linear(config.encoder_ffn_dim, self.embed_dim)
        self.final_layer_norm = _LN(self.embed_dim)

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask, position_embeddings=None, reference_points=None,
                spatial_shapes=None, level_start_index=None, output_attentions=False):
        attn, w = self.self_attn(hidden_states=hidden_states, attention_mask=attention_mask,
                                 encoder_hidden_states=hidden_states, encoder_attention_mask=attention_mask,
                                 position_embeddings=position_embeddings, reference_points=reference_points,
                                 spatial_shapes=spatial_shapes, level_start_index=level_start_index, residual=hidden_states)
        x = self.self_attn_layer_norm(attn)                          # attn already holds hidden_states + attention (epilogue)
        h = ops.linear(x, self.fc1.weight, bias=self.fc1.bias, act=self.act)
        x = self.final_layer_norm(ops.linear(h, self.fc2.weight, bias=self.fc2.bias, residual=x))
        return x, w


class _MHA(nn.MultiheadAttention):
    """nn.MultiheadAttention parameters (in_proj_weight/in_proj_bias/out_proj) with a kernel forward."""

    def run(self, query, key, value, key_lengths=None, key_mask=None, attn_mask=None, residual=None):
        E, H = self.embed_dim, self.num_heads
        B, Tq, _ = query.shape
        Tk = key.shape[1]
        w, b = self.in_proj_weight, self.in_proj_bias
        if query is key:
            qk = ops.linear(query, w[:2 * E], bias=b[:2 * E])
            q, k = qk[..., :E], qk[..., E:]
        else:
            q = ops.linear(query, w[:E], bias=b[:E])
            k = ops.linear(key, w[E:2 * E], bias=b[E:2 * E])
        v = ops.linear(value, w[2 * E:], bias=b[2 * E:])
        ctx = ops.attention(q.unflatten(-1, (H, E // H)), k.unflatten(-1, (H, E // H)),
                            v.unflatten(-1, (H, E // H)), causal=False, seqlens=key_lengths, key_mask=key_mask,
                            attn_mask=attn_mask)
        return ops.linear(ctx, self.out_proj.weight, bias=self.out_proj.bias, residual=residual)


class GroundingDinoDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embed_dim = config.d_model
        self.self_attn = _MHA(self.embed_dim, config.decoder_attention_heads, dropout=config.attention_dropout,
                              batch_first=True)
        self.self_attn_layer_norm = _LN(self.embed_dim)
        self.encoder_attn_text = _MHA(self.embed_dim, config.decoder_attention_heads,
                                      dropout=config.attention_dropout, batch_first=True)
        self.encoder_attn_text_layer_norm = _LN(self.embed_dim)
        self.encoder_attn = GroundingDinoMultiscaleDeformableAttention(
            config, num_heads=config.decoder_attention_heads, n_points=config.decoder_n_points)
        self.encoder_attn_layer_norm = _LN(self.embed_dim)
        self.act = _act(config)
        self.fc1 = nn.Linear(self.embed_dim, config.decoder_ffn_dim)
        self.fc2 = nn.Linear(config.decoder_ffn_dim, self.embed_dim)
        self.final_layer_norm = _LN(self.embed_dim)

    @torch.no_grad()
    def forward(self, hidden_states, position_embeddings=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, vision_encoder_hidden_states=None, vision_encoder_attention_mask=None,
                text_encoder_hidden_states=None, text_encoder_attention_mask=None, self_attn_mask=None,
                output_attentions=False):
        if self_attn_mask is not None:
            raise NotImplementedError("self_attn_mask is only used by contrastive-DN training (:2659-2829)")
        x = hidden_states
        pos = position_embeddings
        qk = x if pos is None else x + pos
        x = self.self_attn_layer_norm(self.self_attn.run(qk, qk, x, residual=x))
        q = x if pos is None else x + pos
        x = self.encoder_attn_text_layer_norm(
            self.encoder_attn_text.run(q, text_encoder_hidden_states, text_encoder_hidden_states,
                                       key_mask=None if text_encoder_attention_mask is None
                                       else ~text_encoder_attention_mask, residual=x))
        attn, _ = self.encoder_attn(hidden_states=x, attention_mask=vision_encoder_attention_mask,
                                    encoder_hidden_states=vision_encoder_hidden_states,
                                    encoder_attention_mask=vision_encoder_attention_mask, position_embeddings=pos,
                                    reference_points=reference_points, spatial_shapes=spatial_shapes,
                                    level_start_index=level_start_index, residual=x)
        x = self.encoder_attn_layer_norm(attn)                       # x + attention, added in the output_proj epilogue
        h = ops.linear(x, self.fc1.weight, bias=self.fc1.bias, act=self.act)
        x = self.final_layer_norm(ops.linear(h, self.fc2.weight, bias=self.fc2.bias, residual=x))
        return (x,)


def get_sine_pos_embed(pos_tensor, num_pos_feats=128, temperature=10000, exchange_xy=True):
    """gd.py:1185-1213: sin/cos features of each coordinate; fp32 like the reference."""
    scale = 2 * math.pi
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=pos_tensor.device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)

    def sine(x):
        sx = x * scale / dim_t
        return torch.stack((sx[..., 0::2].sin(), sx[..., 1::2].cos()), dim=3).flatten(2)

    res = [sine(x) for x in pos_tensor.split([1] * pos_tensor.shape[-1], dim=-1)]
    if exchange_xy:
        res[0], res[1] = res[1], res[0]
    return torch.cat(res, dim=-1)


class GroundingDinoTextEnhancerLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self_attn = _MHA(config.d_model, config.encoder_attention_heads // 2,
                              dropout=getattr(config, "text_enhancer_dropout", 0.0), batch_first=True)
        self.fc1 = nn.Linear(config.d_model, config.encoder_ffn_dim // 2)
        self.fc2 = nn.Linear(config.encoder_ffn_dim // 2, config.d_model)
        self.layer_norm_before = _LN(config.d_model)
        self.layer_norm_after = _LN(config.d_model)
        self.act = _act(config)
        self.num_heads = config.encoder_attention_heads // 2

    @torch.no_grad()
    def forward(self, hidden_states, attention_masks=None, position_embeddings=None):
        """attention_masks: [bs, T, T] bool, True = masked.  Bug-compatible with the reference (gd.py:841-842): it
        expands the mask with ``attention_masks.repeat(num_heads, 1, 1)`` -- batch-minor order -- while
        nn.MultiheadAttention indexes attn_mask as batch*heads + head, so (batch b, head h) uses the mask of batch
        (b*H + h) % bs.  Identical for bs == 1 (the reference's eval setting); reproduced exactly for bs > 1."""
        full = None
        if attention_masks is not None:
            am = attention_masks
            if am.dim() == 3 and am.shape[0] == hidden_states.shape[0]:
                am = am.repeat(self.num_heads, 1, 1)                  # the [bs*H, T, T] tensor MHA receives
            elif am.dim() == 2:
                am = am[None].expand(hidden_states.shape[0] * self.num_heads, -1, -1)
            full = ~am
        qk = hidden_states if position_embeddings is None else hidden_states + position_embeddings
        x = self.layer_norm_before(self.self_attn.run(qk, qk, hidden_states, attn_mask=full, residual=hidden_states))
        h = ops.linear(x, self.fc1.weight, bias=self.fc1.bias, act=self.act)
        x = self.layer_norm_after(ops.linear(h, self.fc2.weight, bias=self.fc2.bias, residual=x))
        return x, None


class GroundingDinoBiMultiHeadAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        vision_dim = text_dim = config.d_model
        self.embed_dim = config.encoder_ffn_dim // 2
        self.num_heads = config.encoder_attention_heads // 2
        self.head_dim = self.embed_dim // self.num_heads
        if self.head_dim * self.num_heads != self.embed_dim:
            raise ValueError("`embed_dim` must be divisible by `num_heads`")
        self.scale = self.head_dim ** (-0.5)
        self.vision_proj = nn.Linear(vision_dim, self.embed_dim)
        self.text_proj = nn.Linear(text_dim, self.embed_dim)
        self.values_vision_proj = nn.Linear(vision_dim, self.embed_dim)
        self.values_text_proj = nn.Linear(text_dim, self.embed_dim)
        self.out_vision_proj = nn.Linear(self.embed_dim, vision_dim)
        self.out_text_proj = nn.Linear(self.embed_dim, text_dim)
        self._packed = None

    def _packed_proj(self):
        ms = (self.vision_proj, self.values_vision_proj, self.text_proj, self.values_text_proj)
        key = tuple((m.weight.data_ptr(), m.weight._version, m.bias._version) for m in ms)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key,
                            torch.cat([ms[0].weight.detach(), ms[1].weight.detach()], 0).contiguous(),
                            torch.cat([ms[0].bias.detach(), ms[1].bias.detach()], 0).contiguous(),
                            torch.cat([ms[2].weight.detach(), ms[3].weight.detach()], 0).contiguous(),
                            torch.cat([ms[2].bias.detach(), ms[3].bias.detach()], 0).contiguous())
        return self._packed[1:]

    @torch.no_grad()
    def forward(self, vision_features, text_features, vision_attention_mask=None, text_attention_mask=None,
                vision_epilogue=None, text_epilogue=None):
        """Both directions share S = (vision_proj(v) * scale) text_proj(t)^T; softmax over text keys gives the
        vision update, softmax over vision keys of S^T the text update (gd.py:927-1004).  The reference's global
        `S - S.max()` and the +-50000 clamp do not change either softmax; masks are True = padded."""
        E, H, D = self.embed_dim, self.num_heads, self.head_dim
        wv, bv, wt, bt = self._packed_proj()
        pv = ops.linear(vision_features, wv, bias=bv)              # [B, S, 2E]: query-side | values
        pt = ops.linear(text_features, wt, bias=bt)                # [B, T, 2E]: key-side | values
        vq, vval = pv[..., :E].unflatten(-1, (H, D)), pv[..., E:].unflatten(-1, (H, D))
        tk, tval = pt[..., :E].unflatten(-1, (H, D)), pt[..., E:].unflatten(-1, (H, D))
        tkm = None if text_attention_mask is None else ~text_attention_mask
        vkm = None if vision_attention_mask is None else ~vision_attention_mask
        v_ctx = ops.attention(vq, tk, tval, scale=self.scale, key_mask=tkm)     # vision queries over text keys
        t_ctx = ops.attention(tk, vq, vval, scale=self.scale, key_mask=vkm)     # text queries over vision keys
        ve = vision_epilogue or {}
        te = text_epilogue or {}
        dv = ops.linear(v_ctx, self.out_vision_proj.weight, bias=self.out_vision_proj.bias, **ve)
        dt = ops.linear(t_ctx, self.out_text_proj.weight, bias=self.out_text_proj.bias, **te)
        return (dv, None), (dt, None)


class GroundingDinoFusionLayer(nn.Module):
    def __init__(self, config, init_values=1e-4):
        super().__init__()
        if getattr(config, "fusion_droppath", 0.0) and False:
            pass
        self.layer_norm_vision = _LN(config.d_model)
        self.layer_norm_text = _LN(config.d_model)
        self.attn = GroundingDinoBiMultiHeadAttention(config)
        self.vision_param = nn.Parameter(init_values * torch.ones((config.d_model)), requires_grad=True)
        self.text_param = nn.Parameter(init_values * torch.ones((config.d_model)), requires_grad=True)

    @torch.no_grad()
    def forward(self, vision_features, text_features, attention_mask_vision=None, attention_mask_text=None):
        v = self.layer_norm_vision(vision_features)
        t = self.layer_norm_text(text_features)
        # residual = the NORMALISED features (gd.py:1092-1099); LayerScale + residual ride in the GEMM epilogue
        (v_new, va), (t_new, ta) = self.attn(v, t, vision_attention_mask=attention_mask_vision,
                                             text_attention_mask=attention_mask_text,
                                             vision_epilogue=dict(colscale=self.vision_param, residual=v),
                                             text_epilogue=dict(colscale=self.text_param, residual=t))
        return (v_new, va), (t_new, ta)


class GroundingDinoEncoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.d_model = config.d_model
        self.text_enhancer_layer = GroundingDinoTextEnhancerLayer(config)
        self.fusion_layer = GroundingDinoFusionLayer(config)
        self.deformable_layer = GroundingDinoDeformableLayer(config)

    def get_text_position_embeddings(self, text_features, text_position_embedding, text_position_ids):
        B, T, _ = text_features.shape
        if text_position_embedding is None and text_position_ids is None:
            pos = torch.arange(T, device=text_features.device).float()[None, :, None].repeat(B, 1, 1)
            text_position_embedding = get_sine_pos_embed(pos, num_pos_feats=self.d_model, exchange_xy=False)
        if text_position_ids is not None:
            text_position_embedding = get_sine_pos_embed(text_position_ids[..., None], num_pos_feats=self.d_model,
                                                         exchange_xy=False)
        return text_position_embedding

    @torch.no_grad()
    def forward(self, vision_features, vision_position_embedding, spatial_shapes, level_start_index, key_padding_mask,
                reference_points, text_features=None, text_attention_mask=None, text_position_embedding=None,
                text_self_attention_masks=None, text_position_ids=None):
        tpos = self.get_text_position_embeddings(text_features, text_position_embedding, text_position_ids).to(
            vision_features.dtype)
        (vision_features, va), (text_features, ta) = self.fusion_layer(
            vision_features=vision_features, text_features=text_features, attention_mask_vision=key_padding_mask,
            attention_mask_text=text_attention_mask)
        text_features, te = self.text_enhancer_layer(hidden_states=text_features,
                                                     attention_masks=~text_self_attention_masks,
                                                     position_embeddings=tpos)
        vision_features, vd = self.deformable_layer(
            hidden_states=vision_features, attention_mask=~key_padding_mask,
            position_embeddings=vision_position_embedding, reference_points=reference_points,
            spatial_shapes=spatial_shapes, level_start_index=level_start_index)
        return (vision_features, text_features), (va, ta, te, vd)
