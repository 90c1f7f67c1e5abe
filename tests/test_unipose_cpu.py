"""CPU: host logic of the H100 UniPose deformable layers (visionllm_b200/unipose.py) against the reference's own
classes (tests/golden/mod_unipose_layers.npz from gen_golden_unipose.py): parameter names, `True = padding` mask
conventions, sequence-first decoder tensors, nn.MultiheadAttention attn_mask / key_padding_mask semantics, 2-d and 4-d
reference points.  Kernels replaced IN THIS TEST ONLY by the fp32 stand-ins of test_gdino_logic_cpu."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from test_gdino_logic_cpu import torch_kernels  # noqa: E402,F401
from unipose_inputs import inputs  # noqa: E402
from weights_util import key_shapes, seeded_state_dict  # noqa: E402


def build():
    from visionllm_b200.unipose import DeformableTransformerDecoderLayer, DeformableTransformerEncoderLayer
    enc = DeformableTransformerEncoderLayer(256, 512, 0.0, "relu", 4, 8, 4).eval()
    enc.load_state_dict(seeded_state_dict(enc, 41))
    dec = DeformableTransformerDecoderLayer(256, 512, 0.0, "relu", 4, 8, 4, use_text_cross_attention=True).eval()
    dec.load_state_dict(seeded_state_dict(dec, 42))
    return enc, dec


def run(enc, dec, x, c=lambda t: t):
    e = enc(c(x["src"]), c(x["pos"]), c(x["ref2"]), x["shapes"], x["lsi"], x["pad"])
    d = dec(tgt=c(x["tgt"]), tgt_query_pos=c(x["qpos"]), tgt_reference_points=c(x["ref4"]),
            memory_text=c(x["memory_text"]), text_attention_mask=x["text_mask"], memory=c(x["memory"]),
            memory_key_padding_mask=x["pad"], memory_level_start_index=x["lsi"], memory_spatial_shapes=x["shapes"],
            self_attn_mask=x["attn_mask"])
    return e, d


def test_unipose_layers_logic_matches_reference(golden_dir, torch_kernels):  # noqa: F811
    g = np.load(os.path.join(golden_dir, "mod_unipose_layers.npz"))
    enc, dec = build()
    assert json.loads(str(g["enc_keys"])) == [list(k) for k in key_shapes(enc)], "encoder-layer keys differ"
    assert json.loads(str(g["dec_keys"])) == [list(k) for k in key_shapes(dec)], "decoder-layer keys differ"
    e, d = run(enc, dec, inputs())
    sub = int(g["sub"])
    for got, ref in ((e[:, ::sub], torch.from_numpy(g["enc_f32"])), (d, torch.from_numpy(g["dec_f32"]))):
        assert got.shape == ref.shape
        assert (got.float() - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item())


# ---- two-stage keypoint decoder (modeling_unipose.py:2869-3130) -------------------------------------------------------
def build_decoder():
    """The H100 decoder built exactly like tests/golden/gen_golden_unipose_decoder.py builds the reference's."""
    import types

    import torch.nn as nn

    import visionllm_b200.unipose as U
    from gen_golden_unipose_decoder import build
    ns = types.SimpleNamespace(DeformableTransformerDecoderLayer=U.DeformableTransformerDecoderLayer,
                               TransformerDecoder=U.TransformerDecoder, MLP=U.MLP, ContrastiveAssign=U.ContrastiveAssign,
                               _LN=U._LN)
    assert nn is not None
    return build(ns)


def decoder_mask(kpt_vis, n_heads, num_body_points):
    from visionllm_b200.unipose import prepare_for_mask
    kpt_mask = torch.cat((torch.ones_like(kpt_vis)[..., 0].unsqueeze(-1), kpt_vis), dim=-1)
    return prepare_for_mask(kpt_mask, n_heads, num_body_points)


def run_decoder(dec, x, mask2, c=lambda t: t):
    text_dict = {"encoded_text": c(x["encoded_text"]), "text_token_mask": ~x["text_mask"]}
    return dec(tgt=c(x["tgt"]).clone(), memory=c(x["memory"]), tgt_mask=None, tgt_mask2=mask2,
               memory_key_padding_mask=x["pad"], pos=None, refpoints_unsigmoid=c(x["ref_unsig"]),
               level_start_index=x["lsi"], spatial_shapes=x["shapes"], valid_ratios=c(x["valid_ratios"]),
               memory_text=c(x["memory_text"]), text_attention_mask=x["text_mask"], text_dict=text_dict,
               kpt_embed=c(x["kpt_embed"]))


def test_unipose_decoder_mask_matches_reference_prepare_for_mask(golden_dir):
    from unipose_inputs import DEC, decoder_inputs
    g = np.load(os.path.join(golden_dir, "mod_unipose_decoder.npz"))
    x = decoder_inputs()
    m = decoder_mask(x["kpt_vis"], DEC["n_heads"], DEC["num_body_points"])
    shp = tuple(int(v) for v in g["mask2_shape"])
    ref = torch.from_numpy(np.unpackbits(g["mask2_bits"], axis=-1)[..., :shp[-1]].astype(bool)).view(shp)
    assert m.dtype == torch.bool and m.shape == (shp[0] * DEC["n_heads"], shp[1], shp[2])
    assert torch.equal(m.view(shp[0], DEC["n_heads"], shp[1], shp[2]), ref[:, None].expand(-1, DEC["n_heads"], -1, -1))


def test_unipose_decoder_logic_matches_reference(golden_dir, torch_kernels):  # noqa: F811
    """Whole decoder loop in fp32 (kernel stand-ins): parameter keys, the top-50 box selection (indices exact), the
    (1 + num_body_points) query expansion, box / keypoint refinement order, every layer's outputs and reference points."""
    from unipose_inputs import DEC, decoder_inputs
    g = np.load(os.path.join(golden_dir, "mod_unipose_decoder.npz"))
    dec, keys = build_decoder()
    assert json.loads(str(g["keys"])) == [list(k) for k in keys], "decoder keys differ"
    x = decoder_inputs()
    mask2 = decoder_mask(x["kpt_vis"], DEC["n_heads"], DEC["num_body_points"])
    hs, refs = run_decoder(dec, x, mask2)
    assert torch.equal(dec.topk_proposals.cpu(), torch.from_numpy(g["topk_f32"])), "top-50 proposal indices differ"
    assert len(hs) == DEC["num_layers"] and len(refs) == DEC["num_layers"] + 1
    rows = stored_rows(g)
    nb = DEC["num_box_decoder_layers"]
    for i, h in enumerate(hs):
        ref = torch.from_numpy(g[f"hs{i}_f32"])
        h = h if i < nb else h[:, rows]
        assert h.shape == ref.shape
        assert (h.float() - ref).abs().max().item() <= 3e-4 * max(1.0, ref.abs().max().item()), i
    for i, r in enumerate(refs):
        ref = torch.from_numpy(g[f"ref{i}_f32"])
        r = r if i - 1 < nb else r[:, rows]
        assert r.shape == ref.shape and (r.float() - ref).abs().max().item() <= 1e-4, i


def stored_rows(g):
    """Expanded-query rows the golden stores (every group_step-th (box + keypoints) group)."""
    from unipose_inputs import DEC
    group, step = DEC["num_body_points"] + 1, int(g["group_step"])
    return torch.cat([torch.arange(gi * group, (gi + 1) * group) for gi in range(0, 50, step)])


# ---- the whole transformer (modeling_unipose.py:2206-2700) ----------------------------------------------------------------
def build_transformer():
    import types

    import visionllm_b200.unipose as U
    from gen_golden_unipose_transformer import build
    ns = types.SimpleNamespace(DeformableTransformer=U.DeformableTransformer, MLP=U.MLP, ContrastiveAssign=U.ContrastiveAssign)
    return build(ns)


def run_transformer(tr, x, mask2, c=lambda t: t):
    from visionllm_b200.unipose import generate_masks_with_text_query_masks
    sa, pid = generate_masks_with_text_query_masks(x["obj_mask"])
    text_dict = {"encoded_text": c(x["encoded_text"]), "text_token_mask": x["obj_mask"].bool(), "position_ids": pid,
                 "text_self_attention_masks": sa}
    return tr([c(s) for s in x["srcs"]], x["masks"], None, [c(p) for p in x["poss"]], None, None, mask2, text_dict, None, None,
              c(x["kpt_embed"]))


def test_text_query_masks_match_reference(golden_dir):
    from unipose_inputs import transformer_inputs
    from visionllm_b200.unipose import generate_masks_with_text_query_masks
    g = np.load(os.path.join(golden_dir, "mod_unipose_transformer.npz"))
    sa, pid = generate_masks_with_text_query_masks(transformer_inputs()["obj_mask"])
    assert torch.equal(sa, torch.from_numpy(g["text_sa"])) and torch.equal(pid, torch.from_numpy(g["text_pid"]))


def test_unipose_transformer_logic_matches_reference(golden_dir, torch_kernels):  # noqa: F811
    """Encoder (fusion + text enhancer + deformable layers), two-stage selection (top-k indices exact), decoder: fp32 logic
    against the reference's own DeformableTransformer."""
    from unipose_inputs import TR, transformer_inputs
    g = np.load(os.path.join(golden_dir, "mod_unipose_transformer.npz"))
    tr, keys = build_transformer()
    assert json.loads(str(g["keys"])) == [list(k) for k in keys], "transformer keys differ"
    x = transformer_inputs()
    mask2 = decoder_mask(x["kpt_vis"], TR["nhead"], TR["num_body_points"])
    hs, refs, hs_enc, ref_enc, init_box = run_transformer(tr, x, mask2)
    assert torch.equal(tr.topk_proposals.cpu(), torch.from_numpy(g["topk_enc"])), "two-stage proposal indices differ"
    assert torch.equal(tr.decoder.topk_proposals.cpu(), torch.from_numpy(g["topk_dec"])), "top-50 box indices differ"
    rows, nb = stored_rows(g), TR["num_box_decoder_layers"]
    for i, h in enumerate(hs):
        ref = torch.from_numpy(g[f"hs{i}_f32"])
        h = h if i < nb else h[:, rows]
        assert h.shape == ref.shape and (h.float() - ref).abs().max().item() <= 5e-4 * max(1.0, ref.abs().max().item()), i
    for i, r in enumerate(refs):
        ref = torch.from_numpy(g[f"ref{i}_f32"])
        r = r if i - 1 < nb else r[:, rows]
        assert r.shape == ref.shape and (r.float() - ref).abs().max().item() <= 2e-4, i
    for got, name in ((hs_enc, "hs_enc"), (ref_enc, "ref_enc"), (init_box, "init_box")):
        ref = torch.from_numpy(g[f"{name}_f32"])
        assert got.shape == ref.shape and (got.float() - ref).abs().max().item() <= 5e-4 * max(1.0, ref.abs().max().item()), name


# ---- the model behind its backbone (modeling_unipose.py:69-655) --------------------------------------------------------------
def build_unipose_model():
    from unipose_inputs import MODEL, TR, transformer_kwargs
    from visionllm_b200.unipose import B200UniPose
    kw = {k: v for k, v in transformer_kwargs().items() if k not in ("d_model", "nhead", "num_queries", "num_feature_levels")}
    m = B200UniPose(hidden_dim=TR["d_model"], l_hidden_size=MODEL["l_hidden"], backbone_channels=MODEL["backbone_channels"],
                    num_feature_levels=TR["num_feature_levels"], num_queries=TR["num_queries"],
                    num_body_points=TR["num_body_points"], num_box_decoder_layers=TR["num_box_decoder_layers"], nheads=TR["nhead"],
                    pe_temperatureH=20, pe_temperatureW=20, **kw).eval()
    m.load_state_dict(seeded_state_dict(m, 71))
    return m


def test_unipose_model_logic_matches_reference_forward(golden_dir, torch_kernels, monkeypatch):  # noqa: F811
    """B200UniPose vs the reference's own `UniPose.forward` (golden): [EMB] projections, input_proj incl. the derived 4th
    level + its sine position embedding, text masks, transformer, box / class / keypoint heads.  fp32 stand-in kernels."""
    import torch.nn.functional as F
    import visionllm_b200.ops as ops
    from unipose_inputs import model_inputs

    def groupnorm_nhwc(x, w, b, groups, eps, relu=False):
        y = F.group_norm(x.float().transpose(1, 2), groups, w.float(), b.float(), eps).transpose(1, 2)
        return torch.relu(y) if relu else y

    monkeypatch.setattr(ops, "groupnorm_nhwc", groupnorm_nhwc)
    g = np.load(os.path.join(golden_dir, "mod_unipose_model.npz"))
    m = build_unipose_model()
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(m)], "model keys differ"
    x = model_inputs()
    out = m(x["feats"], x["poss"], x["text_query"], sample_mask=x["sample_mask"])
    assert torch.equal(m.transformer.topk_proposals, torch.from_numpy(g["topk_enc"]))
    assert torch.equal(m.transformer.decoder.topk_proposals, torch.from_numpy(g["topk_dec"]))
    ref_l = torch.from_numpy(g["logits_f32"])
    assert out.pred_logits.shape == ref_l.shape and torch.equal(torch.isfinite(out.pred_logits), torch.isfinite(ref_l))
    fin = torch.isfinite(ref_l)
    assert (out.pred_logits[fin] - ref_l[fin]).abs().max().item() <= 1e-3 * max(1.0, ref_l[fin].abs().max().item())
    assert (out.pred_boxes - torch.from_numpy(g["boxes_f32"])).abs().max().item() <= 2e-4
    assert (out.pred_keypoints - torch.from_numpy(g["keypoints_f32"])).abs().max().item() <= 2e-4
