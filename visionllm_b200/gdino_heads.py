"""Grounding-DINO query-selection, heads and post-processing of the region/mask decoder (SURVEY 8a a12, a18, a20,
a21), restated from visionllmv2/model/grounding_dino/modeling_ov_grounding_dino_mask_dn.py and
visionllmv2/eval/eval_det.py.  Dense math runs on the wgmma GEMM; the integer work (top-k, //, %, gathers)
uses the same torch primitives the reference uses so indices -- including tie order -- are identical.

  GroundingDinoMLPPredictionHead        gd.py:3704-3720   (bbox / mask-embed / patch2query MLPs, ReLU epilogues)
  GroundingDinoContrastiveEmbedding     gd.py:1410-1428   (q @ text^T, -inf padding to max_text_len, fp32)
  EncoderOutputProposals                gd.py:2228-2276   (per-pixel proposals, validity, inverse sigmoid, enc_output+LN)
  select_topk_proposals                 gd.py:2503-2534   (two-stage top-k query selection)
  forward_seg_heads                     gd.py:2278-2281   (mask einsum 'bqc,bchw->bqhw' as one GEMM per image)
  patch2query_mean                      gd.py:3138        (MLP over the 4 [EMB] states, mean over them)
  post_process_det_gdino / _instseg_    eval_det.py:18-104 (sigmoid, top-k over Q*K, idx//K, idx%K, box scale, masks)
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import msda, ops


class GroundingDinoMLPPredictionHead(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))

    @torch.no_grad()
    def forward(self, x):
        for i, layer in enumerate(self.layers):
            last = i == self.num_layers - 1
            if last and layer.out_features % 8:
                # bbox head: 4 outputs -- pad the weight rows to 8 so the output pitch is 16 bytes
                n = layer.out_features
                w = torch.zeros((8, layer.in_features), dtype=layer.weight.dtype, device=layer.weight.device)
                b = torch.zeros((8,), dtype=layer.bias.dtype, device=layer.bias.device)
                w[:n], b[:n] = layer.weight, layer.bias
                x = ops.linear(x, w, bias=b)[..., :n]
            else:
                x = ops.linear(x, layer.weight, bias=layer.bias, act=None if last else "relu")
        return x


class GroundingDinoContrastiveEmbedding(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.max_text_len = config.max_text_len

    @torch.no_grad()
    def forward(self, vision_hidden_state, text_hidden_state, text_token_mask):
        B, Q, C = vision_hidden_state.shape
        T = text_hidden_state.shape[1]
        Tp = (T + 7) // 8 * 8
        out = torch.full((B, Q, self.max_text_len), float("-inf"), device=vision_hidden_state.device)   # fp32
        buf = torch.empty((B, Q, Tp), dtype=vision_hidden_state.dtype, device=vision_hidden_state.device)
        for b in range(B):
            ops.linear(vision_hidden_state[b], text_hidden_state[b].contiguous(), out=buf[b, :, :T])
        logits = buf[..., :T].masked_fill(~text_token_mask[:, None, :], float("-inf"))
        out[..., :T] = logits
        return out


_GRID_CACHE = {}


@torch.no_grad()
def gen_encoder_output_proposals(enc_output_linear, enc_output_norm, enc_output, padding_mask, spatial_shapes):
    """OVGroundingDinoModel.gen_encoder_output_proposals (gd.py:2228-2276): one (cx, cy, w, h) proposal per pixel,
    validity window (0.01, 0.99), inverse sigmoid with +inf for padded / invalid pixels, zeroed features through
    enc_output + enc_output_norm."""
    B = enc_output.shape[0]
    dev = enc_output.device
    proposals, pos = [], 0
    for level, (H, W) in enumerate(msda.host_shape_list(spatial_shapes)):
        m = padding_mask[:, pos:pos + H * W].view(B, H, W)
        valid_h = (~m[:, :, 0]).sum(1)
        valid_w = (~m[:, 0, :]).sum(1)
        key = (H, W, level, str(dev))
        if key not in _GRID_CACHE:                             # the mask-independent part: (grid + 0.5) and the level's w, h
            gy, gx = torch.meshgrid(torch.linspace(0, H - 1, H, dtype=torch.float32, device=dev),
                                    torch.linspace(0, W - 1, W, dtype=torch.float32, device=dev), indexing="ij")
            grid = torch.stack((gx, gy), -1)[None]
            _GRID_CACHE[key] = (grid + 0.5, torch.ones_like(grid) * 0.05 * (2.0 ** level))
        g05, wh = _GRID_CACHE[key]
        scale = torch.stack((valid_w, valid_h), 1).view(B, 1, 1, 2)
        proposals.append(torch.cat((g05 / scale, wh.expand(B, -1, -1, -1)), -1).view(B, -1, 4))
        pos += H * W
    prop = torch.cat(proposals, 1)
    valid = ((prop > 0.01) & (prop < 0.99)).all(-1, keepdim=True)
    prop = torch.log(prop / (1 - prop))
    # the reference's two masked_fills per tensor (padding, then ~valid) as one pass over the union of the masks
    drop = padding_mask.unsqueeze(-1) | ~valid
    prop = prop.masked_fill(drop, float("inf"))
    q = enc_output.masked_fill(drop, 0.0)
    q = ops.linear(q, enc_output_linear.weight, bias=enc_output_linear.bias)
    q = ops.layernorm(q, enc_output_norm.weight, enc_output_norm.bias, enc_output_norm.eps)
    return q, prop


class EncoderOutputProposals(nn.Module):
    """gen_encoder_output_proposals + enc_output / enc_output_norm (same parameter names as OVGroundingDinoModel)."""

    def __init__(self, d_model):
        super().__init__()
        self.enc_output = nn.Linear(d_model, d_model)
        self.enc_output_norm = nn.LayerNorm(d_model)

    def forward(self, enc_output, padding_mask, spatial_shapes):
        return gen_encoder_output_proposals(self.enc_output, self.enc_output_norm, enc_output, padding_mask, spatial_shapes)


@torch.no_grad()
def select_topk_proposals(enc_outputs_class, enc_outputs_coord_logits, object_query_embedding, num_queries):
    """Two-stage query selection: indices from torch.topk on the per-pixel max class logit (gd.py:2521-2534)."""
    topk_logits = enc_outputs_class.max(-1)[0]
    topk_proposals = torch.topk(topk_logits, num_queries, dim=1)[1]
    coords = torch.gather(enc_outputs_coord_logits, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4))
    cls = torch.gather(enc_outputs_class, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, enc_outputs_class.shape[-1]))
    target = torch.gather(object_query_embedding, 1,
                          topk_proposals.unsqueeze(-1).repeat(1, 1, object_query_embedding.shape[-1]))
    return topk_proposals, coords.sigmoid(), coords, cls, target


@torch.no_grad()
def forward_seg_heads(mask_embed_head, output, mask_features, out_dtype=None):
    """einsum('bqc,bchw->bqhw', mask_embed(output), mask_features) as one [Q,C] x [HW,C]^T GEMM per image.
    out_dtype=torch.float32: the fp32 accumulators are stored directly (the caller's `.float()` as the GEMM's store format,
    like the LLM logits) instead of a bf16 store followed by a widening copy."""
    e = mask_embed_head(output)
    if isinstance(mask_features, tuple):                                  # (rows [B, H*W, C], H, W): the neck's own layout
        f, H, W = mask_features
        B = f.shape[0]
    else:
        B, C, H, W = mask_features.shape
        f = mask_features.permute(0, 2, 3, 1).reshape(B, H * W, C)      # free for channels_last features
        if not f.is_contiguous():
            f = f.contiguous()
    out = torch.empty((B, e.shape[1], H * W), dtype=out_dtype or e.dtype, device=e.device)
    for b in range(B):
        ops.linear(e[b].contiguous(), f[b], out=out[b])
    return out.view(B, e.shape[1], H, W)


@torch.no_grad()
def patch2query_mean(patch2query_head, text_query):
    """text_query [bs, n_cls, num_embs, C_llm] -> [bs, n_cls, d_model]: MLP then mean over the [EMB] states."""
    return patch2query_head(text_query).mean(-2)


def box_cxcywh_to_xyxy(x):
    cx, cy, w, h = x.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)


def _sizes_hw(target_sizes, device):
    if torch.is_tensor(target_sizes):
        return target_sizes.to(device=device, dtype=torch.float32)[:, :2].contiguous()
    return torch.tensor([[float(t[0]), float(t[1])] for t in target_sizes], dtype=torch.float32, device=device)


def det_topk_fused(logits, pred_boxes, target_sizes, num_classes, topk):
    """ONE kernel (csrc/postproc.cu `det_topk_kernel`) for eval_det.py:28-46: sigmoid, top-k over the flattened
    (query, class) grid, `//`, `%`, box gather, cxcywh -> xyxy, (w, h, w, h) scale.  Returns scores [B, k] fp32, labels /
    topk_indexes / box_idx [B, k] int64, boxes [B, k, 4] fp32."""
    from . import _lib
    if logits.dtype != torch.float32 or pred_boxes.dtype != torch.float32 or not logits.is_cuda:
        raise RuntimeError("det_topk_fused: logits / pred_boxes must be CUDA fp32 tensors (the stage's head outputs)")
    B, Q, ld = logits.shape
    if logits.stride(2) != 1 or logits.stride(1) != ld or logits.stride(0) != Q * ld:
        logits = logits.contiguous()
    pred_boxes = pred_boxes.contiguous()
    K = min(int(num_classes), ld)
    k = min(int(topk), Q * K)
    dev = logits.device
    scores = torch.empty((B, k), dtype=torch.float32, device=dev)
    idx, box_idx, labels = (torch.empty((B, k), dtype=torch.int64, device=dev) for _ in range(3))
    boxes = torch.empty((B, k, 4), dtype=torch.float32, device=dev)
    sizes = _sizes_hw(target_sizes, dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().vllm_det_postprocess_f32(logits.data_ptr(), pred_boxes.data_ptr(), sizes.data_ptr(), B, Q, K, ld, k,
                                                 scores.data_ptr(), idx.data_ptr(), box_idx.data_ptr(), labels.data_ptr(),
                                                 boxes.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "vllm_det_postprocess_f32")
    return scores, labels, boxes, idx, box_idx


def mask_chain_fused(pred_masks_i, box_idx_i, image_size, target_size, mask_stride=4):
    """ONE kernel (`mask_chain_kernel`) for eval_det.py:88-99 of one image: masks[box_idx] -> x mask_stride bilinear ->
    crop to image_size -> bilinear to target_size -> sigmoid() > 0.5, without the two full-resolution intermediates."""
    from . import _lib
    if pred_masks_i.dtype != torch.float32 or not pred_masks_i.is_cuda or pred_masks_i.dim() != 3:
        raise RuntimeError("mask_chain_fused: pred_masks of one image must be a CUDA fp32 [Q, H, W] tensor")
    m = pred_masks_i.contiguous()
    bi = box_idx_i.to(torch.int64).contiguous()
    Q, H, W = m.shape
    oh, ow = int(target_size[0]), int(target_size[1])
    ch, cw = min(int(image_size[0]), H * mask_stride), min(int(image_size[1]), W * mask_stride)
    out = torch.empty((bi.numel(), oh, ow), dtype=torch.bool, device=m.device)
    with torch.cuda.device(m.device):
        rc = _lib.lib().vllm_mask_postprocess_f32(m.data_ptr(), bi.data_ptr(), bi.numel(), H, W, int(mask_stride), ch, cw, oh,
                                                  ow, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "vllm_mask_postprocess_f32")
    return out


FUSED_POSTPROCESS = True      # CUDA fp32 head outputs with topk <= 1024 take the fused kernels; False = torch primitives


def _can_fuse(logits, pred_boxes, topk):
    return (FUSED_POSTPROCESS and logits.is_cuda and logits.dtype == torch.float32 and pred_boxes.dtype == torch.float32
            and min(int(topk), logits.shape[1] * logits.shape[2]) <= 1024)


@torch.no_grad()
def post_process_det_gdino(logits, pred_boxes, target_sizes, num_classes, threshold=0.0, topk=100):
    """eval_det.py:18-56.  Returns per-image dicts (scores, labels, boxes) plus the raw index tensors."""
    if _can_fuse(logits, pred_boxes, topk):
        scores, labels, boxes, idx, box_idx = det_topk_fused(logits, pred_boxes, target_sizes, num_classes, topk)
        res = []
        for s, l, bx in zip(scores, labels, boxes):
            if threshold > 0.0:                            # the reference's boolean filter (eval_det.py:50-54)
                keep = s > threshold
                s, l, bx = s[keep], l[keep], bx[keep]
            # threshold == 0 (the eval default): sigmoid outputs in (0, 1] all pass except an exact 0, dropped like the reference
            elif bool((s <= 0).any()):
                keep = s > threshold
                s, l, bx = s[keep], l[keep], bx[keep]
            res.append({"scores": s, "labels": l, "boxes": bx})
        return res, idx, box_idx
    logits = logits[:, :, :num_classes]
    B, Q, K = logits.shape
    prob = logits.sigmoid().view(B, -1)
    k = min(topk, prob.size(1))
    scores, idx = torch.topk(prob, k, dim=1)
    box_idx = torch.div(idx, K, rounding_mode="floor")
    labels = idx % K
    boxes = torch.gather(box_cxcywh_to_xyxy(pred_boxes), 1, box_idx.unsqueeze(-1).repeat(1, 1, 4))
    ts = torch.as_tensor(target_sizes, dtype=torch.float32, device=boxes.device)
    img_h, img_w = ts.unbind(1)
    boxes = boxes * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]
    res = []
    for s, l, bx in zip(scores, labels, boxes):
        keep = s > threshold
        res.append({"scores": s[keep], "labels": l[keep], "boxes": bx[keep]})
    return res, idx, box_idx


@torch.no_grad()
def post_process_instseg_gdino(logits, pred_boxes, pred_masks, target_sizes, image_sizes, num_classes=80, topk=100,
                               mask_stride=4):
    """eval_det.py:59-104: per image top-k, box scale, mask 4x bilinear -> crop -> resize -> sigmoid > 0.5."""
    if _can_fuse(logits, pred_boxes, topk) and pred_masks.dtype == torch.float32:
        scores, labels, boxes, idx, box_idx = det_topk_fused(logits, pred_boxes, target_sizes, num_classes, topk)
        return [{"scores": scores[i], "labels": labels[i], "boxes": boxes[i],
                 "masks": mask_chain_fused(pred_masks[i], box_idx[i], image_sizes[i], target_sizes[i], mask_stride),
                 "topk_indexes": idx[i], "topk_boxes": box_idx[i]} for i in range(logits.shape[0])]
    logits = logits[:, :, :num_classes]
    res = []
    for i in range(logits.shape[0]):
        K = logits.shape[-1]
        prob = logits[i].sigmoid().view(-1)
        k = min(topk, prob.size(0))
        scores, idx = torch.topk(prob, k, dim=0)
        box_idx = torch.div(idx, K, rounding_mode="floor")
        labels = idx % K
        ori_h, ori_w = target_sizes[i][:2]
        boxes = box_cxcywh_to_xyxy(pred_boxes[i][box_idx]) * torch.as_tensor(
            [ori_w, ori_h, ori_w, ori_h], dtype=torch.float32, device=pred_boxes.device)[None, :]
        m = pred_masks[i][box_idx]
        H, W = m.shape[-2:]
        m = F.interpolate(m[:, None], size=(H * mask_stride, W * mask_stride), mode="bilinear", align_corners=False)
        m = m[:, :, :image_sizes[i][0], :image_sizes[i][1]]
        m = F.interpolate(m, size=(ori_h, ori_w), mode="bilinear", align_corners=False)[:, 0]
        res.append({"scores": scores, "labels": labels, "boxes": boxes, "masks": m.sigmoid() > 0.5,
                    "topk_indexes": idx, "topk_boxes": box_idx})
    return res


@torch.no_grad()
def post_process_sem_seg(logits, pred_masks, target_sizes, image_sizes, num_classes=150, sem_seg_postprocess_before_inference=True):
    """eval_semseg.py:16-62 (task 'seg'): per image, class probabilities [nq, K] and mask probabilities [nq, h/4, w/4] ->
    4x bilinear -> crop of the padding -> bilinear to the original size -> einsum('qc,qhw->chw') -> argmax over the classes.
    `sem_seg_postprocess_before_inference=False` contracts with the classes first and resizes the K class maps instead
    (the reference's low-memory order).  Returns a list of int64 [H, W] class maps (the reference returns their `.cpu().numpy()`).
    Host-side torch primitives in the reference's order (no fused kernel yet: one image per call at eval time)."""
    if target_sizes is not None and len(logits) != len(target_sizes):
        raise ValueError("Make sure that you pass in as many target sizes as the batch dimension of the logits")
    res = []
    for cls, mask, image_size, target_size in zip(logits, pred_masks, image_sizes, target_sizes):
        prob = cls[..., :num_classes].sigmoid()
        m = mask.sigmoid()
        H, W = m.shape[-2:]
        size = tuple(int(v) for v in target_size[:2])
        if sem_seg_postprocess_before_inference:
            m = F.interpolate(m[:, None], size=(H * 4, W * 4), mode="bilinear", align_corners=False)
            m = m[:, :, :image_size[0], :image_size[1]]
            m = F.interpolate(m, size=size, mode="bilinear", align_corners=False)[:, 0]
            res.append(torch.einsum("qc,qhw->chw", prob, m).argmax(dim=0))
        else:
            m = torch.einsum("qc,qhw->chw", prob, m)
            m = F.interpolate(m[:, None], size=(H * 4, W * 4), mode="bilinear", align_corners=False)
            m = m[:, :, :image_size[0], :image_size[1]]
            m = F.interpolate(m, size=size, mode="bilinear", align_corners=False)[:, 0]
            res.append(m.argmax(dim=0))
    return res

