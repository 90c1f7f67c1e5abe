"""CPU: host logic of the H100 region encoder (visionllm_b200/region_encoder.py) against the reference's own
`RegionEncoder` run (tests/golden/mod_region_encoder.npz): parameter names, patchify-conv row order, the cumulative
`masks_out` across feature levels, the three pooling modes ('grid_sample' with the reference's recorded point draw).
Kernels are replaced IN THIS TEST ONLY by fp32 torch / the MSDA oracle."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from test_gdino_logic_cpu import torch_kernels  # noqa: E402,F401  (fixture: linear / attention / msda stand-ins)
from weights_util import key_shapes, seeded_state_dict  # noqa: E402


def load_case(golden_dir, mode):
    g = np.load(os.path.join(golden_dir, "mod_region_encoder.npz"))
    cfg = json.loads(str(g["cfg"]))
    feats = [torch.from_numpy(g[f"feat_{i}"]) for i in range(3)]
    if mode == "cross_attn":
        feats = feats[:1]
    B = g["images"].shape[0]
    pts = None
    if mode == "grid_sample":
        pts = [[torch.from_numpy(g[f"points_{lv}_{i}"]) for i in range(B)] for lv in range(3)]
    return g, cfg, feats, pts


@pytest.mark.parametrize("mode", ["mean", "cross_attn", "grid_sample"])
def test_region_encoder_logic_matches_reference(golden_dir, torch_kernels, monkeypatch, mode):  # noqa: F811
    import visionllm_b200.ops as ops
    from visionllm_b200.region_encoder import B200RegionEncoder

    def layernorm(x, w, b, eps, out=None, gelu=False, residual=None):
        y = F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps)
        return F.gelu(y) if gelu else y
    monkeypatch.setattr(ops, "layernorm", layernorm)
    g, cfg, feats, pts = load_case(golden_dir, mode)
    m = B200RegionEncoder(mask_pool_type=mode, **cfg).eval()
    assert json.loads(str(g[f"keys_{mode}"])) == [list(k) for k in key_shapes(m)], "state-dict keys differ"
    m.load_state_dict(seeded_state_dict(m, 77))
    out = m(torch.from_numpy(g["images"]), torch.from_numpy(g["masks"]), feats, sample_points=pts)
    ref = torch.from_numpy(g[f"out_f32_{mode}"])
    assert out.shape == ref.shape
    assert (out.float() - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item())


def test_rand_sample_contract():
    """The restated sampler: rows are (mask id, y/H, x/W) of non-zero pixels, at most max_len, sorted, no repeats."""
    from visionllm_b200.region_encoder import rand_sample
    m = torch.zeros(1, 20, 30)
    m[0, 3:9, 4:14] = 1
    div = torch.tensor([1, 20, 30])[None]
    p = rand_sample(m, div, 25)
    assert p.shape == (25, 3) and (p[:, 0] == 0).all()
    ys, xs = (p[:, 1] * 20).round().long(), (p[:, 2] * 30).round().long()
    assert (m[0, ys, xs] == 1).all() and len({(int(a), int(b)) for a, b in zip(ys, xs)}) == 25
    assert rand_sample(torch.zeros(1, 4, 4), div, 5).shape == (0, 3)
    assert rand_sample(m, div, 10 ** 6).shape == (60, 3)
