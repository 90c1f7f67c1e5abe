"""CPU: host logic of UniPose's image backbone on the H100 modules (visionllm_b200/unipose_backbone.py: reference
parameter names, patch-embed / window / merge padding, shift masks, relative-position bias slabs, out-index norms, mask
interpolation, sine position embedding) against the reference's own `Joiner(SwinTransformer, PositionEmbeddingSineHW)`
(tests/golden/mod_unipose_backbone.npz from gen_golden_unipose_backbone.py).  Kernels replaced IN THIS TEST ONLY by the
fp32 stand-ins of test_gdino_logic_cpu."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from test_gdino_logic_cpu import torch_kernels  # noqa: E402,F401
from unipose_inputs import BACKBONE, backbone_inputs  # noqa: E402
from weights_util import key_shapes, seeded_state_dict  # noqa: E402


def build_joiner():
    from visionllm_b200.unipose_backbone import build_backbone
    c = BACKBONE
    j = build_backbone("swin_T_224_1k", return_interm_indices=c["out_indices"], hidden_dim=c["hidden_dim"],
                       embed_dim=c["embed_dim"], depths=c["depths"], num_heads=c["num_heads"], window_size=c["window_size"]).eval()
    j.load_state_dict(seeded_state_dict(j, 53))
    return j


def test_unipose_backbone_logic_matches_reference(golden_dir, torch_kernels):  # noqa: F811
    g = np.load(os.path.join(golden_dir, "mod_unipose_backbone.npz"))
    j = build_joiner()
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(j)], "Joiner state-dict keys differ from the reference's"
    assert j.num_channels == [128, 256, 512]
    x, mask = backbone_inputs()
    feats, poss = j(x, mask)
    assert len(feats) == len(poss) == 3
    for i, ((t, m), p) in enumerate(zip(feats, poss)):
        ref = torch.from_numpy(g[f"map{i}_f32"])
        assert t.shape == ref.shape
        assert (t.float() - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item()), i
        assert m.dtype == torch.bool and torch.equal(m, torch.from_numpy(g[f"mask{i}"])), i        # masks exact
        assert (p.float() - torch.from_numpy(g[f"pos{i}_f32"])).abs().max().item() <= 1e-5, i


def test_presets_carry_the_reference_table():
    from visionllm_b200.unipose_backbone import SWIN_PRESETS, build_backbone
    assert SWIN_PRESETS["swin_L_384_22k"] == dict(embed_dim=192, depths=[2, 2, 18, 2], num_heads=[6, 12, 24, 48], window_size=12)
    with torch.device("meta"):
        j = build_backbone("swin_T_224_1k")
    assert j.num_channels == [192, 384, 768]                                                        # B200UniPose's default input_proj widths
    keys = set(j.state_dict().keys())
    for k in ("0.patch_embed.proj.weight", "0.patch_embed.norm.bias", "0.layers.0.blocks.1.attn.relative_position_bias_table",
              "0.layers.0.blocks.1.attn.relative_position_index", "0.layers.2.blocks.5.mlp.fc2.weight",
              "0.layers.2.downsample.reduction.weight", "0.norm1.weight", "0.norm3.bias"):
        assert k in keys, k
    assert "0.norm0.weight" not in keys and "0.layers.3.downsample.norm.weight" not in keys
    with pytest.raises(NotImplementedError):
        build_backbone("resnet50")


def test_unipose_model_runs_from_pixels(torch_kernels, monkeypatch):  # noqa: F811
    """B200UniPose(backbone=...).forward_samples == forward() on the backbone's own outputs (the reference's :430 wiring),
    and the state dict carries the backbone under `backbone.0.` like the reference model."""
    import torch.nn.functional as F
    import visionllm_b200.ops as ops
    from unipose_inputs import MODEL, TR, model_inputs, transformer_kwargs
    from visionllm_b200.unipose import B200UniPose

    def groupnorm_nhwc(x, w, b, groups, eps, relu=False):
        y = F.group_norm(x.float().transpose(1, 2), groups, w.float(), b.float(), eps).transpose(1, 2)
        return torch.relu(y) if relu else y

    monkeypatch.setattr(ops, "groupnorm_nhwc", groupnorm_nhwc)
    j = build_joiner()
    kw = transformer_kwargs()
    for k in ("d_model", "nhead", "num_queries", "num_feature_levels"):
        kw.pop(k)
    m = B200UniPose(hidden_dim=TR["d_model"], l_hidden_size=MODEL["l_hidden"], backbone_channels=tuple(j.num_channels),
                    num_feature_levels=4, num_queries=TR["num_queries"], num_body_points=TR["num_body_points"],
                    num_box_decoder_layers=TR["num_box_decoder_layers"], nheads=TR["nhead"], backbone=j, **kw).eval()
    sd = seeded_state_dict(m, 5)
    m.load_state_dict(sd)
    assert any(k.startswith("backbone.0.layers.0.blocks.0.attn.qkv") for k in sd)
    x, mask = backbone_inputs()
    tq = model_inputs()["text_query"]
    a = m.forward_samples(x, mask, tq)
    feats, poss = j(x, mask)
    b = m(feats, poss, tq, sample_mask=mask)
    assert torch.equal(a.pred_boxes, b.pred_boxes) and torch.equal(a.pred_keypoints, b.pred_keypoints)
    assert a.pred_boxes.shape == (2, 50, 4) or a.pred_boxes.shape[0] == 2
    assert torch.isfinite(a.pred_boxes).all()


def test_composite_pose_branch_runs_the_real_unipose(torch_kernels, monkeypatch):  # noqa: F811
    """The composite forward's 'pose' branch (mv2.py:795-836) with the REAL B200UniPose behind it (backbone from pixels,
    transformer, heads; stand-in kernels): the [EMB] hidden states of the LLM reach UniPose as object / keypoint queries and
    the result equals calling UniPose directly on the queries the reference's loop would build."""
    import torch.nn as nn
    import torch.nn.functional as F
    from types import SimpleNamespace
    import visionllm_b200.ops as ops
    from unipose_inputs import TR, transformer_kwargs
    from visionllm_b200.modeling import B200VisionLLMv2Model, pad_images_aug
    from visionllm_b200.unipose import B200UniPose

    def groupnorm_nhwc(x, w, b, groups, eps, relu=False):
        y = F.group_norm(x.float().transpose(1, 2), groups, w.float(), b.float(), eps).transpose(1, 2)
        return torch.relu(y) if relu else y

    monkeypatch.setattr(ops, "groupnorm_nhwc", groupnorm_nhwc)
    C, V = 16, 64

    class FakeViT(nn.Module):
        config = SimpleNamespace(hidden_size=C, patch_size=2)

        def forward(self, x, output_hidden_states=True):
            t = torch.zeros(x.shape[0], 5, C)
            return SimpleNamespace(hidden_states=(t, t, t))

    class FakeLLM(nn.Module):
        def __init__(self):
            super().__init__()
            self.config = SimpleNamespace(hidden_size=C, vocab_size=V)
            self.emb = nn.Embedding(V, C)
            self.dtype = torch.float32

        def get_input_embeddings(self):
            return self.emb

        def forward(self, attention_mask=None, inputs_embeds=None, output_hidden_states=True):
            h = torch.tanh(inputs_embeds) * 2.0
            return SimpleNamespace(hidden_states=(inputs_embeds, h), logits=None)

    j = build_joiner()
    kw = transformer_kwargs()
    for k in ("d_model", "nhead", "num_queries", "num_feature_levels"):
        kw.pop(k)
    torch.manual_seed(11)
    pose = B200UniPose(hidden_dim=TR["d_model"], l_hidden_size=C, backbone_channels=tuple(j.num_channels), num_feature_levels=4,
                       num_queries=TR["num_queries"], num_body_points=TR["num_body_points"],
                       num_box_decoder_layers=TR["num_box_decoder_layers"], nheads=TR["nhead"], backbone=j, **kw).eval()
    pose.load_state_dict(seeded_state_dict(pose, 5))
    cfg = SimpleNamespace(use_pixelshuffle=False, vl_bridge_type="linear", vis_output_layer=-1, num_embs=4, imp_token_id=40,
                          emb_token_id=45, det_tool_id=-1, seg_tool_id=-1, grd_tool_id=-1, pose_tool_id=51)
    m = B200VisionLLMv2Model(cfg, FakeViT(), FakeLLM(), unipose=pose).eval()
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, 30, (2, 48), generator=g)
    n_patch, n_obj = [4, 3], [1, 1]                                   # 1 object class + 3 / 2 keypoint classes
    for b, n in enumerate(n_patch):
        for q in range(n):
            p = 2 + 5 * q
            ids[b, p] = 51
            ids[b, p + 1:p + 5] = 45
    aug = [torch.randn(3, 100, 138, generator=g), torch.randn(3, 80, 110, generator=g)]
    metas = [{"task": "pose", "id2index": {0: 0}} for _ in n_obj]
    out = m(input_ids=ids, images_aug=aug, img_metas=metas)
    up = out.unipose_outputs
    assert up.pred_boxes.shape[0] == 2 and up.pred_keypoints.shape[-1] == TR["num_body_points"] * 3
    assert torch.isfinite(up.pred_boxes).all() and torch.isfinite(up.pred_keypoints).all()
    # the reference's query construction (mv2.py:803-823) on the same hidden states, then UniPose called directly
    h, new_ids = out.last_hidden_state, out.input_ids
    sel = (new_ids >= 45) & (new_ids <= 48)
    obj, kpt = torch.zeros(2, 100, 4, C), torch.zeros(2, 100, 4, C)
    objm, kptm = torch.zeros(2, 100, dtype=torch.bool), torch.zeros(2, 100, dtype=torch.bool)
    for b in range(2):
        tq_i = h[b, sel[b]].reshape(-1, 4, C)
        no, nk = n_obj[b], tq_i.shape[0] - n_obj[b]
        obj[b, :no], objm[b, :no], kpt[b, :nk], kptm[b, :nk] = tq_i[:no], True, tq_i[no:], True
    tensors, mask = pad_images_aug(aug, 32, return_mask=True)
    direct = pose.forward_samples(tensors, mask, dict(obj_querys=obj, obj_query_masks=objm, kpt_querys=kpt, kpt_query_masks=kptm))
    assert torch.equal(direct.pred_boxes, up.pred_boxes) and torch.equal(direct.pred_keypoints, up.pred_keypoints)
    assert torch.equal(torch.isfinite(direct.pred_logits), torch.isfinite(up.pred_logits))
