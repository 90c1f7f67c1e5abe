"""Composite forward: B200 drop-in for ``VisionLLMv2Model.forward`` on the perception / chat eval path.

Restates visionllmv2/model/modeling_visionllmv2.py (paths relative to the VisionLLMv2/ directory of the reference):
  :119-198  constructor-injected sub-models (vis_encoder, llm, gdino) and the vl_bridge variants
  :381-392  pixel_shuffle (space-to-depth x2)
  :419-527  [EMB] super-link injection after tool tokens (overwrite form used by train/eval batches)
  :559-605  ViT -> hidden_states[vis_output_layer][:, 1:] -> pixel shuffle -> vl_bridge -> scatter into
            the <im_patch> positions
  :724-738  llm(inputs_embeds, output_hidden_states=True) -> hidden_states[-1], fp32 logits
  :769-791  [EMB] hidden states -> text_query / text_query_masks -> gdino(...)
Integer index work (token positions, scatter/gather indices) is vectorised but produces the same
indices as the reference's python loops; it is checked index-for-index in tests/test_modeling_cpu.py.
"""
import re
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Optional, Tuple

import torch
import torch.nn as nn
from transformers.utils import ModelOutput

from . import ops


@dataclass
class VisionLLMv2ModelOutput(ModelOutput):
    """Field for field the reference's output class (modeling_visionllmv2.py:57-79): the CausalLMOutputWithPast part
    plus the atom-tool outputs.  Extra read-only conveniences of this drop-in come after the reference's fields."""
    loss: Optional[torch.FloatTensor] = None
    logits: Optional[torch.FloatTensor] = None
    past_key_values: Optional[Tuple[Tuple[torch.FloatTensor]]] = None
    hidden_states: Optional[Tuple[torch.FloatTensor]] = None
    attentions: Optional[Tuple[torch.FloatTensor]] = None
    loss_gdino: Optional[torch.FloatTensor] = None
    gdino_outputs: Any = None
    loss_unipose: Optional[torch.FloatTensor] = None
    unipose_outputs: Any = None
    loss_sd: Optional[torch.FloatTensor] = None
    sd_outputs: Any = None
    loss_ip2p: Optional[torch.FloatTensor] = None
    ip2p_outputs: Any = None
    last_hidden_state: Optional[torch.FloatTensor] = None      # == hidden_states[-1]
    input_ids: Optional[torch.LongTensor] = None               # the ids with the [EMB] slots rewritten (mv2.py:447-468)
    vit_outputs: Any = None


class BridgeLinear(nn.Linear):
    """nn.Linear whose forward is the wgmma GEMM (optionally with a fused activation)."""

    def forward(self, x, act=None):
        return ops.linear(x, self.weight, bias=self.bias, act=act)


class BridgeLayerNorm(nn.LayerNorm):
    def forward(self, x):
        return ops.layernorm(x, self.weight, self.bias, self.eps)


class VLBridge(nn.Sequential):
    """Same module indices / state-dict keys as the reference nn.Sequential (mv2.py:162-184); GELU modules
    are kept as placeholders (so indices match) and fused into the preceding GEMM's epilogue."""

    def forward(self, x, start=0):
        mods = list(self)
        i = start
        while i < len(mods):
            m = mods[i]
            if isinstance(m, BridgeLinear):
                fuse = i + 1 < len(mods) and isinstance(mods[i + 1], nn.GELU)
                x = m(x, act="gelu" if fuse else None)
                i += 2 if fuse else 1
            else:
                x = m(x)
                i += 1
        return x


def build_vl_bridge(vl_bridge_type, v_hidden, l_hidden):
    if vl_bridge_type == "linear":
        return BridgeLinear(v_hidden, l_hidden)          # a bare nn.Linear in the reference: keys `vl_bridge.weight/bias`
    if vl_bridge_type in ("internvl_mlp", "internvl"):
        return VLBridge(BridgeLayerNorm(v_hidden), BridgeLinear(v_hidden, l_hidden), nn.GELU(),
                        BridgeLinear(l_hidden, l_hidden))
    m = re.match(r"^mlp(\d+)x_gelu*", vl_bridge_type)
    if not m:
        raise NotImplementedError(f"{vl_bridge_type} not supported yet.")
    mods = [BridgeLinear(v_hidden, l_hidden)]
    for _ in range(1, int(m.group(1))):
        mods += [nn.GELU(), BridgeLinear(l_hidden, l_hidden)]
    return VLBridge(*mods)


def pixel_shuffle(x, scale_factor=0.5):
    """mv2.py:381-392, verbatim semantics: [n, w, h, c] -> [n, w/2, h/2, 4c]."""
    n, w, h, c = x.size()
    x = x.view(n, w, int(h * scale_factor), int(c / scale_factor))
    x = x.permute(0, 2, 1, 3).contiguous()
    x = x.view(n, int(h * scale_factor), int(w * scale_factor), int(c / (scale_factor * scale_factor)))
    return x.permute(0, 2, 1, 3).contiguous()


def emb_overwrite_indices(input_ids, tool_ids, num_embs):
    """Flat positions (b, p+1+j) that follow a tool token in `tool_ids` -- the slots the reference overwrites
    with the [EMB] ids / embeddings (mv2.py:447-468 with gap_len == num_embs).  Returns (batch_idx, pos_idx, j)."""
    is_tool = torch.zeros_like(input_ids, dtype=torch.bool)
    for t in tool_ids:
        is_tool |= input_ids == t
    b, p = torch.nonzero(is_tool, as_tuple=True)
    j = torch.arange(num_embs, device=input_ids.device)
    pos = p[:, None] + 1 + j[None, :]
    return b[:, None].expand_as(pos).reshape(-1), pos.reshape(-1), j[None, :].expand_as(pos).reshape(-1)


# CUDA bf16 batches take the sequence-assembly kernels (csrc/seqglue.cu) instead of the vectorised torch indexing below;
# both produce the same ids / embeddings / text_query (tests/test_seqglue_gpu.py).  The torch form stays as the host
# logic that the CPU tests pin against the reference's python loops.
FUSED_SEQUENCE = True

IGNORE_INDEX = -100                                                                         # visionllmv2/constant.py:7
GDINO_TASKS = ("det", "det_cap", "grd", "seg", "count_text", "count_visual", "interactive", "ic_mask")   # mv2.py:763


def pad_images_aug(images_aug, size_divisibility=32, return_mask=False):
    """`nested_tensor_from_tensor_list(images_aug, size_divisibility=32).tensors` (util/misc.py:288-316, called at
    mv2.py:771): every [3k, H, W] entry is split into 3-channel images, the batch is zero-padded bottom/right to the
    per-axis maximum rounded UP to a multiple of `size_divisibility`.  (The GDINO caller discards the NestedTensor's own
    mask -- mv2.py:773 re-derives pixel_mask from the red channel; the UniPose caller, mv2.py:798, keeps it:
    `return_mask=True` also returns `.mask` [n, H, W] bool, True = padding, util/misc.py:310-313.)"""
    if torch.is_tensor(images_aug):
        if images_aug.ndim != 4:
            raise ValueError("not supported")
        images_aug = list(images_aug)
    imgs = [piece for t in images_aug for piece in t.split(3, dim=0)]
    if imgs[0].ndim != 3:
        raise ValueError("not supported")
    c = max(im.shape[0] for im in imgs)
    h = max(im.shape[1] for im in imgs)
    w = max(im.shape[2] for im in imgs)
    if size_divisibility > 1:
        h = (h + size_divisibility - 1) // size_divisibility * size_divisibility
        w = (w + size_divisibility - 1) // size_divisibility * size_divisibility
    mask = None
    if return_mask:
        mask = torch.ones((len(imgs), h, w), dtype=torch.bool, device=imgs[0].device)
        for im, m in zip(imgs, mask):
            m[: im.shape[1], : im.shape[2]] = False
    if all(tuple(im.shape) == (c, h, w) for im in imgs):
        out = torch.stack(imgs)
    else:
        out = torch.zeros((len(imgs), c, h, w), dtype=imgs[0].dtype, device=imgs[0].device)
        for im, dst in zip(imgs, out):
            dst[: im.shape[0], : im.shape[1], : im.shape[2]].copy_(im)
    return (out, mask) if return_mask else out


def pose_text_query(text_query, text_query_masks, num_patches, num_objcls, max_obj=100, max_kpt=100):
    """mv2.py:801-831: split every sample's [EMB] patches into its first `num_objcls[b]` object-class patches and the
    remaining keypoint patches, zero-padded to 100 slots each.  `text_query` [bs, mx, num_embs, C] / `text_query_masks`
    [bs, mx] are the per-sample patch lists the GDINO branch also builds (same rows of `hidden_states`); `num_patches`
    and `num_objcls` are host ints (len(img_metas[b]['id2index'])).  A sample with no object class or no keypoint keeps
    all-zero queries and masks (the reference's `if num_objcls != 0 and num_kpts != 0`)."""
    bs, _, n_emb, C = text_query.shape
    obj = text_query.new_zeros((bs, max_obj, n_emb, C))
    kpt = text_query.new_zeros((bs, max_kpt, n_emb, C))
    obj_m = torch.zeros((bs, max_obj), dtype=torch.bool, device=text_query.device)
    kpt_m = torch.zeros((bs, max_kpt), dtype=torch.bool, device=text_query.device)
    for b in range(bs):
        no, nk = int(num_objcls[b]), int(num_patches[b]) - int(num_objcls[b])
        if no != 0 and nk != 0:
            if no > max_obj or nk > max_kpt or nk < 0:
                raise ValueError(f"sample {b}: {no} object-class / {nk} keypoint [EMB] patches do not fit the reference's "
                                 f"{max_obj} / {max_kpt} slots (mv2.py:806-809)")
            obj[b, :no], obj_m[b, :no] = text_query[b, :no], True
            kpt[b, :nk], kpt_m[b, :nk] = text_query[b, no:no + nk], True
    return dict(obj_querys=obj, obj_query_masks=obj_m, kpt_querys=kpt, kpt_query_masks=kpt_m)


def region_encoder_inputs(images, regions, vit_hidden_states, split_sizes, num_splits=None):
    """The tensors the reference hands its region encoder (mv2.py:609-687), vectorised: every region of a sample is
    paired with the sample's GLOBAL view -- the image itself ('pad': `images` a [bs,3,h,w] tensor), the last tile
    ('anyres': a list of [n_tiles,3,h,w]), or, for multi-image in-context samples (`num_splits`: per sample the tile
    count of each image), the last tile of the r-th image for the r-th region -- and with the patch tokens (CLS
    dropped) of that view in the last three ViT hidden states.

    regions: list of [n_region_i, h, w] 0/1 masks.  Returns (all_images [R,3,h,w], all_regions [R,1,h,w],
    [3 x all_image_features [R, n_tokens, C]])."""
    num_regions = [len(r) for r in regions]
    all_regions = torch.cat([r[:, None] for r in regions], dim=0)
    dev = all_regions.device
    if torch.is_tensor(images):                                     # 'pad': one view per sample, row b of the ViT batch
        view_rows = [torch.full((n,), b, dtype=torch.long, device=dev) for b, n in enumerate(num_regions)]
        flat_images = images
    else:
        images = [x.unsqueeze(0) if x.ndim == 3 else x for x in images]
        sizes = split_sizes if split_sizes is not None else [im.shape[0] for im in images]
        starts = [0]
        for n in sizes[:-1]:
            starts.append(starts[-1] + n)
        view_rows = []
        for b, n in enumerate(num_regions):
            if num_splits is not None:                              # r-th region <-> last tile of the r-th image
                ends, acc = [], 0
                for k in num_splits[b]:
                    acc += k
                    ends.append(acc - 1)
                rows = torch.as_tensor(ends[:n], dtype=torch.long, device=dev) + starts[b]
                if len(rows) != n:
                    raise RuntimeError("mmic sample with more regions than images (mv2.py:634 would mis-pair them)")
            else:                                                   # all regions <-> the last (global) tile
                rows = torch.full((n,), starts[b] + sizes[b] - 1, dtype=torch.long, device=dev)
            view_rows.append(rows)
        flat_images = torch.cat(list(images), dim=0)
    rows = torch.cat(view_rows) if view_rows else torch.zeros(0, dtype=torch.long, device=dev)
    all_images = flat_images[rows]
    feats = [h[rows, 1:] for h in vit_hidden_states[-3:]]
    return all_images, all_regions, feats


def scatter_region_tokens(input_ids, inputs_embeds, region_features, reg_token_id):
    """mv2.py:690-698: the k-th `<region>` token of the flattened batch takes the k-th region feature."""
    B, L, C = inputs_embeds.shape
    mask = (input_ids == reg_token_id).reshape(-1)
    if int(mask.sum()) != region_features.shape[0]:
        raise RuntimeError(f"{int(mask.sum())} <region> tokens vs {region_features.shape[0]} region features")
    flat = inputs_embeds.reshape(B * L, C).clone()
    flat[mask] = region_features.to(flat.dtype)
    return flat.reshape(B, L, C)


class B200VisionLLMv2Model(nn.Module):
    def __init__(self, config, vis_encoder, llm, gdino=None, region_encoder=None, unipose=None):
        super().__init__()
        self.config = config
        self.vis_encoder = vis_encoder
        self.llm = llm
        self.use_pixelshuffle = bool(getattr(config, "use_pixelshuffle", False))
        self.v_hidden_size = vis_encoder.config.hidden_size
        self.l_hidden_size = llm.config.hidden_size
        vh = self.v_hidden_size * 4 if self.use_pixelshuffle else self.v_hidden_size
        self.vl_bridge = build_vl_bridge(getattr(config, "vl_bridge_type", "linear"), vh, self.l_hidden_size)
        self.use_gdino = gdino is not None
        if gdino is not None:
            self.gdino = gdino
        self.use_region_encoder = region_encoder is not None
        if region_encoder is not None:
            self.region_encoder = region_encoder
        self.use_unipose = unipose is not None                         # a B200UniPose built with backbone= (mv2.py:795-836)
        if unipose is not None:
            self.unipose = unipose
        self.num_embs = int(getattr(config, "num_embs", 4))
        self.emb_embeddings_det = nn.Embedding(self.num_embs, self.l_hidden_size)
        self.emb_embeddings_pose = nn.Embedding(self.num_embs, self.l_hidden_size)
        # special-token ids are assigned by init_special_token_ids (mv2.py:281-353)
        for k in ("imp_token_id", "emb_token_id", "det_tool_id", "seg_tool_id", "grd_tool_id", "pose_tool_id",
                  "reg_token_id"):
            setattr(self, k, getattr(config, k, -1))

    # ---- pieces ------------------------------------------------------------------------------
    def inject_emb(self, input_ids, inputs_embeds):
        """[EMB] ids/embeddings after det/seg/grd (and pose) tool tokens -- overwrite form."""
        ids, emb = input_ids.clone(), inputs_embeds
        L = ids.shape[1]
        for tools, table in (((self.det_tool_id, self.seg_tool_id, self.grd_tool_id), self.emb_embeddings_det),
                             ((self.pose_tool_id,), self.emb_embeddings_pose)):
            tools = [t for t in tools if t is not None and t >= 0]
            if not tools:
                continue
            b, p, j = emb_overwrite_indices(ids, tools, self.num_embs)
            if b.numel() == 0:
                continue
            # The reference takes the overwrite form (gap_len == num_embs) only when [EMB] ids are already present in
            # the FIRST row (mv2.py:426-431); otherwise it INSERTS (gap_len == 0, generation).  Refuse instead of
            # clobbering real tokens: every target slot must already hold an [EMB] id.
            in_range = p < L
            slots = ids[b[in_range], p[in_range]]
            ok = bool(in_range.all()) and bool(((slots >= self.emb_token_id)
                                                & (slots < self.emb_token_id + self.num_embs)).all())
            if not ok:
                if self.uses_insert_form(input_ids):
                    return self.inject_emb_insert(input_ids, inputs_embeds)
                raise NotImplementedError("a tool token without its pre-placed [EMB] slots in a batch whose first row carries "
                                          "[EMB] ids: the reference's overwrite form (mv2.py:430-431) would clobber real tokens")
            ids[b, p] = self.emb_token_id + j
            emb = emb.clone() if emb is inputs_embeds else emb
            emb[b, p] = table.weight.to(emb.dtype)[j]
        return ids, emb

    def _tool_groups(self):
        return (((self.det_tool_id, self.seg_tool_id, self.grd_tool_id), self.emb_embeddings_det),
                ((self.pose_tool_id,), self.emb_embeddings_pose))

    def uses_insert_form(self, input_ids):
        """mv2.py:425-431: the reference inspects the FIRST row only -- a tool token there and no `emb_token_id` means
        gap_len = 0 (the [EMB] ids / embeddings are INSERTED after every tool token: generation, multi-round chat history)."""
        row = input_ids[0]
        tools = [t for grp, _ in self._tool_groups() for t in grp if t is not None and t >= 0]
        has_tool = any(bool((row == t).any()) for t in tools)
        return has_tool and not bool((row == self.emb_token_id).any())

    def inject_emb_insert(self, input_ids, inputs_embeds):
        """The gap_len == 0 form of mv2.py:436-527: after every det / seg / grd (then pose) tool token the `num_embs` [EMB] ids
        and the tool's emb_embeddings are inserted; the sequence grows.  Restated with the reference's own order of operations,
        including its quirk: the insertion points are the positions found in the ORIGINAL row and are not shifted by earlier
        insertions of the same row (so a second tool token's [EMB] block lands `num_embs` tokens early, exactly as in the
        reference).  Rows must end up equally long (the reference `torch.stack`s them)."""
        emb_ids = torch.arange(self.emb_token_id, self.emb_token_id + self.num_embs, dtype=torch.long, device=input_ids.device)
        new_ids, new_emb = [], []
        for row_ids, row_emb in zip(input_ids, inputs_embeds):
            ids, emb = row_ids, row_emb
            for tools, table in self._tool_groups():
                pos = torch.cat([torch.where(row_ids == t)[0] for t in tools if t is not None and t >= 0] or
                                [row_ids.new_zeros((0,))])
                block = table.weight.to(row_emb.dtype)
                for p0 in pos.tolist():
                    ids = torch.cat((ids[:p0 + 1], emb_ids, ids[p0 + 1:]), 0)
                    emb = torch.cat((emb[:p0 + 1], block, emb[p0 + 1:]), 0)
            new_ids.append(ids)
            new_emb.append(emb)
        if len({t.shape[0] for t in new_ids}) != 1:
            raise RuntimeError("rows carry different numbers of tool tokens: the reference cannot stack them either (mv2.py:526)")
        return torch.stack(new_ids, 0), torch.stack(new_emb, 0)

    def encode_images(self, images):
        if isinstance(images, (list, tuple)):                      # 'anyres': bs x [1 + n_split, 3, h, w]
            images = [x.unsqueeze(0) if x.ndim == 3 else x for x in images]
            split_sizes = [im.shape[0] for im in images]
            concat = torch.cat(list(images), dim=0)
        else:
            split_sizes, concat = None, images
        outs = self.vis_encoder(concat, output_hidden_states=True)
        hs = outs.hidden_states[getattr(self.config, "vis_output_layer", -2)]
        if (self.use_pixelshuffle and FUSED_SEQUENCE and hs.is_cuda and hs.dtype == torch.bfloat16
                and self.llm.dtype == torch.bfloat16 and hs.stride(2) == 1):
            # CLS slice + pixel shuffle (+ the LayerNorm that opens internvl_mlp) in ONE pass: the projector's A operand
            mods = list(self.vl_bridge) if isinstance(self.vl_bridge, VLBridge) else None
            if mods and isinstance(mods[0], BridgeLayerNorm):
                x = ops.pixel_shuffle_rows(hs, 1, mods[0].weight, mods[0].bias, mods[0].eps)
                return self.vl_bridge(x, start=1), split_sizes, outs
            return self.vl_bridge(ops.pixel_shuffle_rows(hs, 1)), split_sizes, outs
        feats = hs[:, 1:].to(self.llm.dtype)
        if self.use_pixelshuffle:
            h = w = int(feats.shape[1] ** 0.5)
            feats = pixel_shuffle(feats.reshape(feats.shape[0], h, w, -1), 0.5)
            feats = feats.reshape(feats.shape[0], -1, feats.shape[-1])
        return self.vl_bridge(feats), split_sizes, outs

    def scatter_image_tokens(self, input_ids, inputs_embeds, image_features, split_sizes):
        B, L, C = inputs_embeds.shape
        selected = input_ids == self.imp_token_id
        has_image = selected.sum(-1) != 0
        if split_sizes is not None:
            has_image = torch.repeat_interleave(has_image, torch.tensor(split_sizes, device=has_image.device))
        vit_embeds = image_features[has_image].reshape(-1, C)
        flat = inputs_embeds.reshape(B * L, C).clone()
        sel = selected.reshape(-1)
        n_sel = int(sel.sum())
        if n_sel != vit_embeds.shape[0]:
            raise RuntimeError(f"image token count mismatch: {n_sel} <im_patch> slots vs {vit_embeds.shape[0]} "
                               "ViT tokens (the reference tiles/trims and zeroes the loss here, mv2.py:591-604; "
                               "this drop-in refuses instead of guessing)")
        flat[sel] = vit_embeds.to(flat.dtype)
        return flat.reshape(B, L, C)

    def gather_text_query(self, input_ids, hidden_states):
        """mv2.py:776-787: [EMB] hidden states -> text_query [bs, max_cls, num_embs, C], masks [bs, max_cls]."""
        B, L, C = hidden_states.shape
        emb_select = (input_ids >= self.emb_token_id) & (input_ids <= self.emb_token_id + self.num_embs - 1)
        counts = emb_select.sum(-1)
        if int(counts.sum()) == 0:
            return None, None
        num_patches = counts // self.num_embs
        mx = int(num_patches.max())
        tq = torch.zeros((B, mx, self.num_embs, C), dtype=hidden_states.dtype, device=hidden_states.device)
        tm = torch.zeros((B, mx), dtype=torch.bool, device=hidden_states.device)
        b, p = torch.nonzero(emb_select, as_tuple=True)
        rank = torch.cumsum(emb_select.int(), -1)[b, p] - 1          # order of the [EMB] token within its row
        keep = rank < (num_patches * self.num_embs)[b]
        b, p, rank = b[keep], p[keep], rank[keep]
        tq.view(B, mx * self.num_embs, C)[b, rank] = hidden_states[b, p]
        tm[b, rank // self.num_embs] = True
        return tq, tm

    # ---- forward -------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, input_ids=None, inputs_embeds=None, attention_mask=None, images=None, images_aug=None,
                img_metas=None, targets=None, labels=None, past_key_values=None, use_cache=False,
                output_attentions=False, output_hidden_states=False, return_dict=True, regions=None, num_splits=None,
                region_sample_points=None, logits_rows=None, **unused):
        if past_key_values is not None or use_cache:
            raise NotImplementedError("generation with KV cache is outside the forward hot path")
        if targets is not None:
            raise NotImplementedError("detection / pose training losses (matcher, criterion, denoising queries) are outside "
                                      "the forward hot path (SURVEY 8f)")
        if labels is not None and logits_rows is not None:
            raise ValueError("labels need the logits of every position: do not pass logits_rows together with labels")
        embed_w = self.llm.get_input_embeddings().weight
        fused = (FUSED_SEQUENCE and input_ids is not None and input_ids.is_cuda and embed_w.dtype == torch.bfloat16
                 and (inputs_embeds is None or (inputs_embeds.dtype == torch.bfloat16 and inputs_embeds.is_contiguous())))
        vit_out, plan, feats, split_sizes = None, None, None, False
        if images is not None:
            feats, split_sizes, vit_out = self.encode_images(images)
        if fused:
            plan = ops.seq_index(input_ids, (self.det_tool_id, self.seg_tool_id, self.grd_tool_id), (self.pose_tool_id,),
                                 self.emb_token_id, self.num_embs, self.imp_token_id,
                                 split_sizes if images is not None else False, feats.shape[1] if feats is not None else 0)
            status = int(plan.status.item())
            if status & 1:
                # no pre-placed [EMB] slots: the reference's insert form (mv2.py:428-429) changes the sequence length -- host
                # logic of the torch path below (inject_emb decides between inserting and refusing)
                fused, plan = False, None
            elif status & 2:
                raise RuntimeError("image token count mismatch between the <im_patch> slots and the ViT tokens (the "
                                   "reference tiles/trims and zeroes the loss here, mv2.py:591-604; this drop-in refuses)")
        if fused:
            inputs_embeds = ops.assemble_embeds(
                plan, embed_w, self.emb_embeddings_det.weight, self.emb_embeddings_pose.weight,
                feats.reshape(-1, feats.shape[-1]).contiguous() if feats is not None else None, base_embeds=inputs_embeds)
            input_ids = plan.new_ids
        else:
            if inputs_embeds is None:
                inputs_embeds = self.llm.get_input_embeddings()(input_ids)
            input_ids, inputs_embeds = self.inject_emb(input_ids, inputs_embeds)
            if images is not None:
                inputs_embeds = self.scatter_image_tokens(input_ids, inputs_embeds, feats.to(inputs_embeds.dtype),
                                                          split_sizes)
        if attention_mask is not None and attention_mask.shape[1] != input_ids.shape[1]:    # mv2.py:539-545 (after an insertion)
            add = input_ids.shape[1] - attention_mask.shape[1]
            if add < 0:
                raise ValueError("attention_mask is longer than the sequence")
            attention_mask = torch.cat((attention_mask, attention_mask.new_ones((attention_mask.shape[0], add))), -1)
        if images is not None:
            if self.use_region_encoder and regions is not None:                              # mv2.py:607-698
                ri, rm, rf = region_encoder_inputs(images, regions, vit_out.hidden_states, split_sizes, num_splits)
                rfeat = self.region_encoder(ri, rm, rf, sample_points=region_sample_points)
                inputs_embeds = scatter_region_tokens(input_ids, inputs_embeds, rfeat, self.reg_token_id)
        # logits_rows (extension): lm_head on those flattened [B*L] positions only -> out.logits is fp32 [n, V]
        head_kw = {} if logits_rows is None else {"logits_rows": logits_rows}
        out = self.llm(attention_mask=attention_mask, inputs_embeds=inputs_embeds, output_hidden_states=True, **head_kw)
        hidden = out.hidden_states[-1]
        loss = None
        if labels is not None:                                                               # mv2.py:740-757
            # the reference masks the [EMB] slots of the CALLER's labels in place (:743-744); so does this drop-in
            labels[(labels >= self.emb_token_id) & (labels <= self.emb_token_id + self.num_embs - 1)] = IGNORE_INDEX
            # "shift so that tokens < n predict n": rather than slicing the fp32 logits (a 1.5 GB copy at cfg 3), shift the
            # labels and ignore each row's last position -- the same (logit row, label) pairs, the same mean
            shift = torch.cat((labels[:, 1:], torch.full_like(labels[:, :1], IGNORE_INDEX)), 1).to(out.logits.device)
            lg = out.logits
            loss = ops.ce_loss(lg.reshape(-1, lg.shape[-1]), shift.reshape(-1))
        gdino_outputs, unipose_outputs = None, None
        task = img_metas[0]["task"] if img_metas is not None else None                       # mv2.py:755-758
        if task == "pose" and images_aug is not None and not self.use_unipose:
            raise NotImplementedError("task 'pose' routes the [EMB] states to UniPose (mv2.py:795-836): build the composite "
                                      "with unipose=B200UniPose(..., backbone=build_backbone(...))")
        # mv2.py:762-763: the region decoder runs only for these tasks (no img_metas -> task None -> no gdino_outputs)
        if self.use_gdino and images_aug is not None and task in GDINO_TASKS:
            if plan is not None and hidden.dtype == torch.bfloat16 and hidden.is_contiguous():
                mx = int((plan.emb_count // self.num_embs).max()) if plan.B else 0
                tq, tm = ops.text_query_gather(plan, hidden, self.num_embs, mx) if mx > 0 else (None, None)
            else:
                tq, tm = self.gather_text_query(input_ids, hidden)
            if tq is not None:
                pixel_values = pad_images_aug(images_aug, 32)                               # mv2.py:771-772
                pixel_mask = pixel_values[:, 0, :, :] != 0                                  # mv2.py:773
                gdino_outputs = self.gdino(pixel_values, pixel_mask=pixel_mask, text_query=tq,
                                           text_query_masks=tm, img_metas=img_metas, labels=None)
        if self.use_unipose and task == "pose" and images_aug is not None:                   # mv2.py:795-836
            if plan is not None and hidden.dtype == torch.bfloat16 and hidden.is_contiguous():
                n_patch = (plan.emb_count // self.num_embs).tolist() if plan.B else []
                mx = max(n_patch) if n_patch else 0
                tq, tm = ops.text_query_gather(plan, hidden, self.num_embs, mx) if mx > 0 else (None, None)
            else:
                tq, tm = self.gather_text_query(input_ids, hidden)
                n_patch = tm.sum(-1).tolist() if tm is not None else []
            if tq is not None:                                                               # "if have [EMB] tokens" (:801)
                tensors, pad_mask = pad_images_aug(images_aug, 32, return_mask=True)         # :798
                n_obj = [len(m["id2index"]) for m in img_metas]                              # :812
                unipose_outputs = self.unipose.forward_samples(tensors, pad_mask,
                                                               pose_text_query(tq, tm, n_patch, n_obj))
        if not return_dict:                                                                  # mv2.py:873-875
            output = (out.logits,) + (None, out.hidden_states, None)
            return (loss,) + output if loss is not None else output
        return VisionLLMv2ModelOutput(loss=loss, logits=out.logits, past_key_values=None, hidden_states=out.hidden_states,
                                      attentions=None, gdino_outputs=gdino_outputs, unipose_outputs=unipose_outputs,
                                      last_hidden_state=hidden, vit_outputs=vit_out, input_ids=input_ids)
