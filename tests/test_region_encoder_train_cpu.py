"""CPU: the host logic of region-encoder training (visionllm_b200/train.py region_encoder_train: patch rows, K padding,
differentiable conv-weight views, the per-level point tables, the level accumulation and mean) with fp32 torch stand-ins
for the kernels' autograd Functions, against the reference RegionEncoder's fp32 gradients
(tests/golden/train_region_encoder.npz); and the refusals that need no device."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from weights_util import key_shapes, seeded_state_dict  # noqa: E402


class _Linear:
    @staticmethod
    def apply(x, w, out_f32=False, residual=None, bias=None):
        return F.linear(x, w, bias)


class _LayerNormGelu:
    @staticmethod
    def apply(x, w, b, eps):
        return F.gelu(F.layer_norm(x, (x.shape[-1],), w, b, eps))


class _RegionPool:
    """masks_out accumulates the levels; each level pools its point table (bilinear, zero padding, weights, / count)."""

    @staticmethod
    def apply(emb, enc, feats, tables):
        masks_out, pooled = emb, []
        for f, (loc, wgt) in zip(feats, tables):
            masks_out = masks_out + f
            grid = (loc * 2 - 1).unsqueeze(2)                                           # [R, n, 1, 2]
            s = F.grid_sample(masks_out.permute(0, 3, 1, 2), grid, align_corners=False)[..., 0].transpose(1, 2)
            pooled.append(((s * wgt[..., None]).sum(1) / wgt.sum(1, keepdim=True)).nan_to_num())
        return torch.stack(pooled)


def test_host_logic_matches_reference_gradients(golden_dir, monkeypatch):
    from visionllm_b200 import train
    from visionllm_b200.region_encoder import B200RegionEncoder
    monkeypatch.setattr(train, "LinearFn", _Linear)
    monkeypatch.setattr(train, "LayerNormGeluFn", _LayerNormGelu)
    monkeypatch.setattr(train, "RegionPoolFn", _RegionPool)
    gz = np.load(os.path.join(golden_dir, "train_region_encoder.npz"))
    m = B200RegionEncoder(mask_pool_type="grid_sample", **json.loads(str(gz["cfg"])))
    assert json.loads(str(gz["keys"])) == [list(k) for k in key_shapes(m)]
    m.load_state_dict(seeded_state_dict(m, 77))
    B = gz["images"].shape[0]
    pts = [[torch.from_numpy(gz[f"points_{lv}_{i}"]) for i in range(B)] for lv in range(3)]
    assert min(len(p) for p in pts[0]) < 16                          # a region with less than one query group
    out = train.region_encoder_train(m, torch.from_numpy(gz["images"]), torch.from_numpy(gz["masks"]),
                                     [torch.from_numpy(gz[f"feat_{i}"]) for i in range(3)], sample_points=pts)
    ref = torch.from_numpy(gz["out_f32"])
    assert float((out.detach() - ref).norm() / ref.norm()) <= 1e-4
    out.backward(torch.from_numpy(gz["grad_out"]))
    named = dict(m.named_parameters())
    for n in json.loads(str(gz["params"])):
        r = torch.from_numpy(gz[f"grad_f32/{n}"])
        err = float((named[n].grad - r).norm() / r.norm())
        assert err <= 1e-4, (n, err)


def test_refusals_before_any_kernel():
    from test_padded_training_cpu import _composite
    from visionllm_b200.region_encoder import B200RegionEncoder
    from visionllm_b200.train import B200VisionLLMv2ModelTrain, region_encoder_train
    for mode in ("mean", "cross_attn"):
        enc = B200RegionEncoder(64, 256, 96, mask_pool_type=mode)
        with pytest.raises(NotImplementedError, match="grid_sample"):
            region_encoder_train(enc, torch.zeros(1, 3, 112, 112), torch.zeros(1, 1, 112, 112), [])
    m = _composite()
    tr = B200VisionLLMv2ModelTrain(m)
    ids = torch.randint(0, 30, (2, 8))
    with pytest.raises(NotImplementedError, match="without a region encoder"):
        tr(input_ids=ids, regions=[torch.ones(1, 8, 8)])
    m.region_encoder, m.use_region_encoder = B200RegionEncoder(64, 256, 96, mask_pool_type="mean"), True
    with pytest.raises(NotImplementedError, match="grid_sample"):
        tr(input_ids=ids, regions=[torch.ones(1, 8, 8)])
