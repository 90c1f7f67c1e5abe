"""CPU: the whole Grounding-DINO stage -- backbone, neck, encoder, mask FPN, two-stage selection, decoder, heads -- of
`visionllm_b200.gdino_model.B200GroundingDinoForObjectDetection` against the REFERENCE'S OWN
`OVGroundingDinoForObjectDetection.forward_test` on CPU in fp32, same state dict.  The reference's outputs and its
state-dict keys are stored goldens (tests/golden/gen_golden_gdino_model_cpu.py ran the reference on the weights and
inputs that the functions below rebuild from their seeds).  Kernels are replaced by fp32 torch stand-ins in this test
only (no GPU here); this pins the host logic: layouts, masks, valid ratios, reference points, top-k selection, box
refinement, head wiring, parameter names."""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from test_gdino_logic_cpu import torch_kernels  # noqa: E402,F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
STAGE_CASES = [(False, False), (True, False), (True, True)]          # (ragged padding masks, our Swin backbone)


def stage_kwargs(b200_backbone):
    from transformers import SwinConfig
    bc = SwinConfig(image_size=64, embed_dim=32 if b200_backbone else 24, depths=[1, 2, 1, 1], num_heads=[1, 2, 4, 8], window_size=4,
                    out_features=["stage1", "stage2", "stage3", "stage4"])
    return dict(backbone_config=bc, d_model=256, encoder_layers=2, decoder_layers=2, encoder_ffn_dim=256, decoder_ffn_dim=256,
                num_queries=20, num_feature_levels=4, dropout=0., attention_dropout=0., activation_dropout=0.,
                mask_dim=256, norm="GN", l_hidden_size=64)


def internimage_kwargs():
    # H width (the reference hard-codes the neck's input widths to 320..2560, gd.py:5183), one layer per level
    bc = dict(model_type="internimage-H", core_op="DCNv3_pytorch", depths=[1, 1, 1, 1], level2_post_norm_block_ids=[0],
              with_cp=False)
    return dict(backbone_config=bc, d_model=256, encoder_layers=1, decoder_layers=1, encoder_ffn_dim=256, decoder_ffn_dim=256,
                num_queries=12, num_feature_levels=4, dropout=0., attention_dropout=0., activation_dropout=0.,
                mask_dim=256, norm="GN", l_hidden_size=64)


def stage_golden(ragged, b200_backbone):
    return f"gdino_cpu_stage_{'ragged' if ragged else 'full'}_{'b200swin' if b200_backbone else 'hfswin'}.npz"


def stage_state_dict(module, seed):
    from weights_util import seeded_state_dict
    sd = seeded_state_dict(module, seed)
    for k in sd:                                                  # LayerScale-style gates: make the fusion path count
        if k.endswith("vision_param") or k.endswith("text_param"):
            sd[k] = sd[k] * 0 + 0.5
    return sd


def stage_inputs(ragged, l_hidden=64):
    g = torch.Generator().manual_seed(5)
    B, Hh, W = 2, 128, 160
    x = torch.randn(B, 3, Hh, W, generator=g)
    pm = torch.ones(B, Hh, W, dtype=torch.long)
    if ragged:
        pm[1, 96:, :] = 0
        pm[1, :, 120:] = 0
    tq = torch.randn(B, 5, 4, l_hidden, generator=g)
    tm = torch.ones(B, 5, dtype=torch.bool)
    tm[1, 3:] = False
    return x, pm, tq, tm


def neck_inputs(l_hidden=64):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 3, 100, 136, generator=g)
    pm = torch.ones(1, 100, 136, dtype=torch.long)
    pm[0, 80:] = 0
    return x, pm, torch.randn(1, 3, 4, l_hidden, generator=g), torch.ones(1, 3, dtype=torch.bool)


def internimage_inputs(l_hidden=64):
    g = torch.Generator().manual_seed(6)
    B, Hh, W = 2, 64, 96
    x = torch.randn(B, 3, Hh, W, generator=g)
    pm = torch.ones(B, Hh, W, dtype=torch.long)
    pm[1, 32:, :] = 0
    return x, pm, torch.randn(B, 4, 4, l_hidden, generator=g), torch.ones(B, 4, dtype=torch.bool)


def build_ours(kw, seed, golden, b200_backbone=False):
    """Our stage on the seeded state dict; the golden records the reference's state-dict keys / shapes."""
    from weights_util import key_shapes
    from visionllm_b200.gdino_model import B200GroundingDinoForObjectDetection
    from visionllm_b200.swin import B200SwinBackbone
    cfg = SimpleNamespace(encoder_attention_heads=8, decoder_attention_heads=8, encoder_n_points=4, decoder_n_points=4,
                          activation_function="relu", max_text_len=256, query_dim=4, two_stage=True,
                          embedding_init_target=True, two_stage_bbox_embed_share=False, decoder_bbox_embed_share=True,
                          position_embedding_type="sine", positional_embedding_temperature=20, **kw)
    ours = B200GroundingDinoForObjectDetection(
        cfg, backbone_model=B200SwinBackbone(cfg.backbone_config) if b200_backbone else None).eval()
    # identical parameter names and shapes
    assert json.loads(str(golden["keys"])) == [list(k) for k in key_shapes(ours)]
    ours.load_state_dict(stage_state_dict(ours, seed))
    return cfg, ours


@pytest.fixture()
def gn_kernel(monkeypatch, torch_kernels):  # noqa: F811
    import visionllm_b200.ops as ops

    from oracle import torch_kernels as TK

    monkeypatch.setattr(ops, "groupnorm_nhwc", TK.groupnorm_nhwc)
    monkeypatch.setattr(ops, "conv2d_s1_rows", TK.conv2d_s1_rows)
    monkeypatch.setattr(ops, "upsample_add_nhwc", TK.upsample_add_nhwc)


def check_outputs(b, g):
    logits, boxes, masks = (torch.from_numpy(g[k]) for k in ("logits", "pred_boxes", "pred_masks"))
    assert logits.shape == b.logits.shape and masks.shape == b.pred_masks.shape
    finite = torch.isfinite(logits)
    assert torch.equal(finite, torch.isfinite(b.logits))                      # -inf padding pattern identical
    assert (logits[finite] - b.logits[finite]).abs().max() < 2e-3
    assert (boxes - b.pred_boxes).abs().max() < 1e-4
    assert (masks - b.pred_masks).abs().max() < 2e-2 * masks.abs().max().clamp(min=1)


@pytest.mark.parametrize("ragged,b200_backbone", STAGE_CASES)
def test_whole_stage_matches_reference_forward_test(gn_kernel, ragged, b200_backbone):
    g = np.load(os.path.join(GOLDEN, stage_golden(ragged, b200_backbone)))
    cfg, ours = build_ours(stage_kwargs(b200_backbone), 11, g, b200_backbone)
    x, pm, tq, tm = stage_inputs(ragged)
    with torch.no_grad():
        b = ours.forward_test(x, pixel_mask=pm, text_query=tq, text_query_masks=tm)
    check_outputs(b, g)


def test_neck_integer_outputs_match_reference(gn_kernel):
    """spatial_shapes / level_start_index (int64) exactly; valid_ratios, masks exactly (same torch ops): what the
    reference's neck hands to its encoder (captured at the encoder call when the golden was made)."""
    g = np.load(os.path.join(GOLDEN, "gdino_cpu_neck.npz"))
    cfg, ours = build_ours(stage_kwargs(False), 12, g)
    x, pm, tq, tm = neck_inputs()
    with torch.no_grad():
        feats = ours.model.backbone_features(x)
        src, mflat, pos, shapes, lsi, vr = ours.model.neck(feats, pm)
    cap = {k: torch.from_numpy(g[k]) for k in g.files if k != "keys"}
    assert torch.equal(shapes, cap["spatial_shapes"]) and shapes.dtype == torch.int64
    assert torch.equal(lsi, cap["level_start_index"])
    assert torch.equal(~mflat, cap["vision_attention_mask"])
    assert torch.equal(vr, cap["valid_ratios"])
    assert (src - cap["vision_features"]).abs().max() < 1e-4
    assert (pos - cap["vision_position_embedding"]).abs().max() < 1e-5


def test_whole_stage_with_internimage_backbone_matches_reference(gn_kernel, monkeypatch):
    """`backbone_config = {'model_type': 'internimage-H', ...}` (gd.py:2073-2074, 5154-5195): the reference builds
    `GroundingDinoInternImageBackbone`, we build `visionllm_b200.internimage` from the same dict; same state dict, same
    forward_test outputs.  The reference ran its pure-PyTorch core op (golden); ours runs the C oracle of the CUDA core."""
    import visionllm_b200.dcnv3 as dcn
    import visionllm_b200.ops as ops
    from oracle import dcnv3_oracle as O

    def layernorm(x, w, b, eps, out=None, gelu=False, residual=None):
        y = F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps)
        if residual is not None:
            y = y + residual.float()
        return F.gelu(y) if gelu else y

    def dwconv_nhwc(x, wt, bias, k):
        C = x.shape[-1]
        return F.conv2d(x.float().permute(0, 3, 1, 2), wt.float().t().reshape(C, 1, k, k), bias.float(), padding=k // 2,
                        groups=C).permute(0, 2, 3, 1).contiguous()

    def dcnv3_prep(packed, G, K, with_scale):
        lead = packed.shape[:-1]
        mask = F.softmax(packed[..., G * K * 2:G * K * 3].reshape(*lead, G, K), -1).reshape(*lead, G * K).contiguous()
        return (packed[..., :G * K * 2].contiguous(), mask,
                packed[..., G * K * 3:G * K * 3 + G].sigmoid() if with_scale else None)

    def dcnv3_blend(core, xproj, scale, gc):
        if scale is None:
            return core
        s_ = scale[..., None].expand(*scale.shape, gc).reshape(core.shape)
        return core * (1 - s_) + xproj * s_

    def dcnv3_forward(inp, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, gc, offset_scale, step=256, **kw_):
        return torch.from_numpy(np.asarray(O.forward(inp.float().numpy(), offset.float().numpy(), mask.float().numpy(),
                                                     kh, kw, sh, sw, ph, pw, dh, dw, group, gc, offset_scale),
                                           dtype=np.float32))

    for name, fn in (("layernorm", layernorm), ("dwconv_nhwc", dwconv_nhwc),
                     ("dcnv3_prep", dcnv3_prep), ("dcnv3_blend", dcnv3_blend)):
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(dcn, "dcnv3_forward", dcnv3_forward)

    g = np.load(os.path.join(GOLDEN, "gdino_cpu_internimage.npz"))
    cfg, ours = build_ours(internimage_kwargs(), 21, g)
    assert type(ours.model.backbone.conv_encoder.model).__name__ == "B200InternImage"
    x, pm, tq, tm = internimage_inputs()
    with torch.no_grad():
        b = ours.forward_test(x, pixel_mask=pm, text_query=tq, text_query_masks=tm)
    check_outputs(b, g)


def test_conv_rows_prepadded_forms_agree(gn_kernel):
    """conv_rows / NormConv2d.rows on the zero-bordered map `upsample_add_nhwc(..., pad=)` writes (the copy-free mask-FPN chain)
    equal the plain call on the unpadded map -- for the implicit-GEMM 3x3 form (border consumed by the convolution) and for
    shapes that take the general path (border dropped again)."""
    import torch.nn as nn
    from visionllm_b200.gdino_model import NormConv2d, conv_rows
    g = torch.Generator().manual_seed(3)
    for C, k, p in ((64, 3, 1), (24, 3, 1), (64, 1, 0)):                 # 3 * 64 % 64 == 0: implicit; 3 * 24: general; 1x1
        x = torch.randn(2, 6, 7, C, generator=g)
        conv = NormConv2d(C, 32, k, padding=p, relu=True).eval()
        nn.init.normal_(conv.weight, std=0.1)
        xp = torch.nn.functional.pad(x, (0, 0, p, p, p, p))
        a, Ha, Wa = conv_rows(x, conv)
        b, Hb, Wb = conv_rows(xp, conv, prepadded=p > 0)
        assert (Ha, Wa) == (Hb, Wb) == (6, 7) and torch.allclose(a, b.reshape(a.shape), atol=1e-6)
        ra, _, _ = conv.rows(x)
        rb, _, _ = conv.rows(xp, prepadded=p > 0)
        assert ra.shape == rb.shape == (2, 42, 32) and torch.allclose(ra, rb, atol=1e-5)
