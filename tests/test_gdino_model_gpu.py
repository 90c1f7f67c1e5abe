"""GPU: the whole Grounding-DINO stage (`B200GroundingDinoForObjectDetection.forward_test`: HF Swin backbone ->
our neck (GEMM + GroupNorm kernel) -> encoder -> mask FPN -> two-stage top-k -> decoder -> heads) against the golden
produced by the REFERENCE's `OVGroundingDinoForObjectDetection.forward_test` (tests/golden/gen_golden_gdino_model.py).

Tolerance (floating point, bf16 compute): rel_l2(ours, ref_fp32) <= 1.5 * rel_l2(ref_bf16, ref_fp32) + 1e-3 -- we may
not be further from the fp32 reference than 1.5x the reference's own bf16 deployment is.  The top-k selection is
discrete: the reference's own bf16 run already selects a different set than its fp32 run on this vector, so tensors
after the selection are compared with the selection pinned to the golden's indices (as the generator does for the
reference's bf16 leg), and the free-running selection is checked for overlap."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))


def rel(a, b):
    m = torch.isfinite(b)
    assert torch.equal(m, torch.isfinite(a))
    return ((a[m] - b[m]).norm() / b[m].norm()).item()


def stage_config():
    from transformers import SwinConfig
    from types import SimpleNamespace
    bc = SwinConfig(image_size=64, embed_dim=32, depths=[2, 2, 2, 2], num_heads=[1, 2, 4, 8], window_size=4,
                    out_features=["stage1", "stage2", "stage3", "stage4"])
    return SimpleNamespace(backbone_config=bc, d_model=256, encoder_layers=2, decoder_layers=2, encoder_ffn_dim=512,
                           decoder_ffn_dim=512, encoder_attention_heads=8, decoder_attention_heads=8, num_queries=20,
                           num_feature_levels=4, encoder_n_points=4, decoder_n_points=4, dropout=0., attention_dropout=0.,
                           activation_dropout=0., activation_function="relu", mask_dim=256, norm="GN", l_hidden_size=64,
                           max_text_len=256, query_dim=4, two_stage=True, embedding_init_target=True,
                           two_stage_bbox_embed_share=False, decoder_bbox_embed_share=True, position_embedding_type="sine",
                           positional_embedding_temperature=20)


@pytest.fixture(scope="module", params=["hf_swin", "b200_swin"])
def stage(golden_dir, request):
    """Backbone either HF's SwinBackbone run by torch (how the reference builds it) or ours on the H100 kernels."""
    from weights_util import key_shapes, seeded_state_dict
    from visionllm_b200.gdino_model import B200GroundingDinoForObjectDetection
    from visionllm_b200.swin import B200SwinBackbone
    g = np.load(os.path.join(golden_dir, "mod_gdino_model.npz"))
    cfg = stage_config()
    m = B200GroundingDinoForObjectDetection(
        cfg, backbone_model=B200SwinBackbone(cfg.backbone_config) if request.param == "b200_swin" else None).eval()
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(m)]          # the reference's state-dict keys
    sd = seeded_state_dict(m, int(g["seed"]))
    for k in sd:
        if k.endswith("vision_param") or k.endswith("text_param"):
            sd[k] = sd[k] * 0 + 0.5
    m.load_state_dict(sd)
    m = m.cuda().bfloat16()
    return m, g


def _inputs(g):
    return (torch.from_numpy(g["pixel_values"]).cuda().bfloat16(), torch.from_numpy(g["pixel_mask"]).cuda(),
            torch.from_numpy(g["text_query"]).cuda().bfloat16(), torch.from_numpy(g["text_query_masks"]).cuda())


def _check(name, ours, g, slack=1.5):
    ref32 = torch.from_numpy(g[name + "_f32"])
    ref16 = torch.from_numpy(g[name + "_refbf16"])
    e_ref = rel(ref16, ref32)
    e = rel(ours.float().cpu().reshape(ref32.shape), ref32)
    assert e <= slack * e_ref + 1e-3, f"{name}: ours {e:.5f} vs reference-bf16 {e_ref:.5f}"
    return e, e_ref


def test_stage_up_to_selection(stage):
    m, g = stage
    x, pm, tq, tm = _inputs(g)
    sub = int(g["sub"])
    o = m.forward_test(x, pixel_mask=pm, text_query=tq, text_query_masks=tm).model_outputs
    mf, Hm, Wm = o.mask_features
    _check("enc_vision", o.encoder_last_hidden_state_vision[:, ::sub], g)
    _check("enc_text", o.encoder_last_hidden_state_text, g)
    _check("mask_features", mf[:, ::sub], g)
    _check("enc_class_max", o.enc_outputs_class.float().max(-1)[0], g, slack=2.0)
    _check("enc_coord", o.enc_outputs_coord_logits[:, ::sub], g)
    # integer side of the neck
    assert o.spatial_shapes.tolist() == [[12, 16], [6, 8], [3, 4], [2, 2]] and o.spatial_shapes.dtype == torch.int64
    assert o.level_start_index.tolist() == [0, 192, 240, 252]
    # free-running selection: indices are torch.topk of OUR logits (exact), and mostly the golden's
    mine = torch.topk(o.enc_outputs_class.max(-1)[0], 20, dim=1)[1]
    assert torch.equal(mine, o.topk_proposals)
    gold = torch.from_numpy(g["topk"]).cuda()
    overlap = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(mine, gold)) / gold.numel()
    assert overlap >= 0.8, overlap


def test_stage_after_selection_with_pinned_topk(stage, monkeypatch):
    import visionllm_b200.gdino_heads as H
    m, g = stage
    x, pm, tq, tm = _inputs(g)
    gold = torch.from_numpy(g["topk"]).cuda()

    def pinned(enc_class, enc_coord, oq, nq):
        coords = torch.gather(enc_coord, 1, gold.unsqueeze(-1).repeat(1, 1, 4))
        cls = torch.gather(enc_class, 1, gold.unsqueeze(-1).repeat(1, 1, enc_class.shape[-1]))
        tgt = torch.gather(oq, 1, gold.unsqueeze(-1).repeat(1, 1, oq.shape[-1]))
        return gold, coords.sigmoid(), coords, cls, tgt

    monkeypatch.setattr(H, "select_topk_proposals", pinned)
    o = m.forward_test(x, pixel_mask=pm, text_query=tq, text_query_masks=tm)
    assert o.logits.dtype == torch.float32 and o.pred_boxes.dtype == torch.float32 and o.pred_masks.dtype == torch.float32
    assert tuple(o.pred_masks.shape) == (2, 20, 24, 32)
    _check("init_ref", o.model_outputs.init_reference_points, g)
    _check("logits", o.logits, g)
    _check("boxes", o.pred_boxes, g)
    _check("masks", o.pred_masks.reshape(2, -1), g)


@pytest.mark.parametrize("shape", [(2, 4096, 256, 32), (3, 777, 256, 32), (1, 65536, 256, 32), (2, 100, 512, 32), (1, 5, 192, 8)])
@pytest.mark.parametrize("relu", [False, True])
def test_groupnorm_kernel(shape, relu):
    """csrc/groupnorm.cu vs torch fp32 GroupNorm of the same bf16 input: one bf16 rounding of the fp32 result."""
    from visionllm_b200 import ops
    N, HW, C, G = shape
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(N, HW, C, device="cuda", generator=g) * 2 + 0.7).bfloat16()
    w = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
    y = ops.groupnorm_nhwc(x, w, b, G, 1e-5, relu=relu)
    ref = torch.nn.functional.group_norm(x.float().transpose(1, 2), G, w.float(), b.float(), 1e-5).transpose(1, 2)
    if relu:
        ref = ref.relu()
    err = (y.float() - ref).abs()
    assert (err <= 2.0 ** -8 * ref.abs() + 1e-4).all(), err.max().item()       # bf16 half-ulp + stats noise
    y2 = ops.groupnorm_nhwc(x, w, b, G, 1e-5, relu=relu)
    assert torch.equal(y, y2)                                                    # deterministic statistics


@pytest.mark.parametrize("shape", [(2, 16, 16, 32, 32, 256), (1, 13, 17, 25, 34, 64), (2, 8, 8, 8, 8, 48), (1, 5, 7, 20, 9, 8)])
def test_upsample_add_kernel_matches_the_torch_ops(shape):
    """vllm_upsample_add_nhwc_bf16 (FPN top-down step) vs the reference's ops: bf16 F.interpolate(bilinear,
    align_corners=False) + bf16 add.  ATen's kernel may contract the tap sums differently, so the interpolated value can
    differ by a bf16 ulp: checked against the fp32 interpolation with one bf16 rounding of each step."""
    from visionllm_b200 import ops
    B, Hi, Wi, Ho, Wo, C = shape
    g = torch.Generator(device="cuda").manual_seed(Hi * Wo)
    top = torch.randn(B, Hi, Wi, C, device="cuda", generator=g).bfloat16()
    lat = torch.randn(B, Ho, Wo, C, device="cuda", generator=g).bfloat16()
    out = ops.upsample_add_nhwc(top, lat)
    up16 = torch.nn.functional.interpolate(top.permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=False)
    ref_ops = lat + up16.permute(0, 2, 3, 1)                                     # the reference's bf16 ops
    up32 = torch.nn.functional.interpolate(top.float().permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear",
                                           align_corners=False).permute(0, 2, 3, 1)
    ref32 = lat.float() + up32
    assert out.shape == lat.shape and out.dtype == torch.bfloat16
    tol = 2.0 ** -7 * ref32.abs() + 2.0 ** -7 * up32.abs() + 1e-6
    assert ((out.float() - ref32).abs() <= tol).all()
    assert (out != ref_ops).float().mean().item() < 0.02                         # bit-equal to the torch ops but for rare ulps


def test_groupnorm_rejects_bad_arguments():
    from visionllm_b200 import ops
    x = torch.zeros(1, 8, 48, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(48, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.groupnorm_nhwc(x, w, w, 12, 1e-5)            # 4 channels per group: not a multiple of 8
    with pytest.raises(RuntimeError):
        ops.groupnorm_nhwc(x.float(), w, w, 2, 1e-5)


def test_cuda_graph_replay_matches_eager(stage):
    """visionllm_b200.graphs.GraphedForward: the whole stage captured into one CUDA graph (no host sync inside the
    forward) replays to exactly the eager result, also after the inputs change."""
    from visionllm_b200.graphs import GraphedForward
    m, g = stage
    x, pm, tq, tm = _inputs(g)
    gf = GraphedForward(lambda a, b, c, d: m.forward_test(a, pixel_mask=b, text_query=c, text_query_masks=d))
    for trial in range(3):
        xi = x if trial == 0 else (x * (1.0 + 0.25 * trial)).contiguous()
        eager = m.forward_test(xi, pixel_mask=pm, text_query=tq, text_query_masks=tm)
        e = [t.clone() for t in (eager.logits, eager.pred_boxes, eager.pred_masks)]
        o = gf(xi, pm, tq, tm)
        for a, b in zip(e, (o.logits, o.pred_boxes, o.pred_masks)):
            assert torch.equal(a, b)
    assert gf.launches_per_replay > 50 and len(gf._cache) == 1


@pytest.mark.parametrize("B,Hh,W,C,Cout,k,p", [(2, 24, 32, 256, 256, 3, 1), (1, 7, 5, 64, 72, 3, 1), (3, 16, 16, 128, 256, 3, 0),
                                               (1, 256, 256, 256, 256, 3, 1), (2, 9, 11, 64, 32, 5, 2)])
def test_implicit_gemm_conv_vs_torch(B, Hh, W, C, Cout, k, p):
    """vllm_conv_rows_bf16 (overlapping-row TMA map over the zero-padded map, K walked in kernel_h shifted segments)
    vs F.conv2d in fp32 on the same bf16 values: one bf16 output rounding."""
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 100 + Hh)
    x = torch.randn(B, Hh, W, C, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, C, k, k, device="cuda", generator=g) / (C * k * k) ** 0.5).bfloat16()
    b = torch.randn(Cout, device="cuda", generator=g).bfloat16()
    y = ops.conv2d_s1_rows(x, w.permute(0, 2, 3, 1).reshape(Cout, -1).contiguous(), b, k, p, act="relu")
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=p).relu().permute(0, 2, 3, 1)
    assert y.shape == ref.shape
    assert ((y.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 2e-3).all(), (y.float() - ref).abs().max().item()


def _torch_sine(feats, dim_t, pre):
    cols = []
    for f in feats:
        e = (f * pre if pre else f)[:, None] / dim_t
        cols.append(torch.stack((e[:, 0::2].sin(), e[:, 1::2].cos()), dim=2).flatten(1))
    return torch.cat(cols, 1)


def test_sine_embed_kernel_matches_the_torch_chain():
    """csrc/posembed.cu vs the reference's elementwise chains evaluated by torch on the same GPU (gd.py:529-564 neck form with
    `.to(bf16) + level_embed` into a level slab of a [B, S, C] buffer; gd.py:1755-1790 decoder form with strided columns):
    same IEEE operations in the same order, so fp32 results agree to the last bit unless the two libdevice builds differ
    (then <= 2 ulp); bf16 results differ on no more than a rounding tie."""
    from visionllm_b200 import ops
    from visionllm_b200.gdino_model import GroundingDinoSinePositionEmbedding
    g = torch.Generator(device="cuda").manual_seed(11)
    # decoder form: proposals [B, Q, L, 4] fp32, level-0 slice, feature order (y, x, w, h), 2 pi pre-scale
    B, Q = 3, 100
    ref_in = torch.rand(B, Q, 4, 4, device="cuda", generator=g)
    p = ref_in[:, :, 0, :]
    d = torch.arange(128, dtype=torch.float32, device="cuda")
    dim_t = 10000 ** (2 * torch.div(d, 2, rounding_mode="floor") / 128)
    want = _torch_sine([p[:, :, c].reshape(-1) for c in (1, 0, 2, 3)], dim_t, 2 * math.pi)
    got = ops.sine_embed([p[:, :, c] for c in (1, 0, 2, 3)], p.stride(1), dim_t, B * Q, pre_scale=2 * math.pi)
    assert got.shape == (B * Q, 512) and got.dtype == torch.float32
    assert (got - want).abs().max().item() <= 2.4e-7 and (got == want).float().mean().item() >= 0.999
    got16 = ops.sine_embed([p[:, :, c] for c in (1, 0, 2, 3)], p.stride(1), dim_t, B * Q, pre_scale=2 * math.pi, out_dtype=torch.bfloat16)
    w16 = want.bfloat16()
    assert (got16 == w16).float().mean().item() >= 0.999 and (got16.float() - w16.float()).abs().max().item() <= 2 ** -7
    # neck form: a padded mask, two levels written into one [B, S, 256] buffer with the level embedding added in bf16
    pe = GroundingDinoSinePositionEmbedding(128, 20, normalize=True)
    lvl = (torch.randn(2, 256, device="cuda", generator=g) * 0.5).bfloat16()
    masks = []
    for (h, w) in ((24, 40), (12, 20)):
        m = torch.ones(2, h, w, dtype=torch.bool, device="cuda")
        m[1, int(h * 0.8):] = False
        m[1, :, int(w * 0.7):] = False
        masks.append(m)
    S = sum(m.shape[1] * m.shape[2] for m in masks)
    buf = torch.full((2, S, 256), 7.0, dtype=torch.bfloat16, device="cuda")
    off = 0
    for i, m in enumerate(masks):
        y, x = pe.embeds(m)
        n = m.shape[1] * m.shape[2]
        ops.sine_embed([y.contiguous(), x.contiguous()], 1, pe.dim_t(m.device), 2 * n, out=buf[:, off:off + n], add_row=lvl[i].contiguous())
        ref = pe(m).to(torch.bfloat16).flatten(1, 2) + lvl[i].view(1, 1, -1)
        got = buf[:, off:off + n]
        assert (got == ref).float().mean().item() >= 0.999, i
        assert (got.float() - ref.float()).abs().max().item() <= 2 ** -6, i
        off += n


@pytest.mark.parametrize("B,H,W,C,k,p", [(2, 24, 32, 256, 3, 1), (1, 7, 5, 64, 3, 1), (2, 9, 11, 64, 5, 2)])
def test_fpn_chain_without_copies_is_bit_identical(B, H, W, C, k, p):
    """The mask-FPN chain in its copy-free form -- upsample_add written into the zero-bordered map (pad=), top read through a
    batch pitch, the 3x3 convolution on the prepadded map, GroupNorm reading the convolution's corner of the padded grid in
    place -- against the same kernels with the copies (F.pad, .contiguous()) in between: identical bits."""
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 10 + H)
    S = (H // 2) * (W // 2) + 37
    flat = torch.randn(B, S, C, device="cuda", generator=g).bfloat16()               # "encoder output": level slab + other levels
    top = flat[:, :(H // 2) * (W // 2)].reshape(B, H // 2, W // 2, C)
    assert not top.is_contiguous() or B == 1
    lat = torch.randn(B, H, W, C, device="cuda", generator=g).bfloat16()
    wt = (torch.randn(C, k * k * C, device="cuda", generator=g) / (C * k * k) ** 0.5).bfloat16()
    gam = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
    bet = (0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
    # with copies
    y0 = ops.upsample_add_nhwc(top.contiguous(), lat)
    c0 = ops.conv2d_s1_rows(y0, wt, None, k, p)
    n0 = ops.groupnorm_nhwc(c0.reshape(B, -1, C), gam, bet, 32 if C % 256 == 0 else 8, 1e-5, relu=True)
    # copy-free
    y1 = ops.upsample_add_nhwc(top, lat, pad=p)
    assert y1.shape == (B, H + 2 * p, W + 2 * p, C)
    assert torch.equal(y1[:, p:H + p, p:W + p], y0)
    border = y1.clone(); border[:, p:H + p, p:W + p] = 0
    assert not border.any()
    c1 = ops.conv2d_s1_rows(y1, wt, None, k, p, prepadded=True)
    assert torch.equal(c1, c0) and not c1.is_contiguous()
    n1 = ops.groupnorm_nhwc(c1, gam, bet, 32 if C % 256 == 0 else 8, 1e-5, relu=True)
    assert n1.is_contiguous() and torch.equal(n1, n0)
