"""GPU: the InternImage backbone on our kernels (SURVEY 8a-a13) -- depthwise conv and LN+GELU kernels against fp32
torch on the same bf16 inputs, and the whole backbone against the reference's own `InternImage` run
(tests/golden/mod_internimage_small.npz) under the module tolerance rule of test_modules_gpu.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from weights_util import key_shapes, seeded_state_dict  # noqa: E402


def rel_l2(a, b):
    return float(torch.linalg.norm(a.float() - b.float()) / torch.linalg.norm(b.float()))


@pytest.mark.parametrize("k,shape", [(5, (2, 17, 23, 64)), (3, (1, 8, 5, 320)), (7, (2, 9, 12, 16)), (5, (1, 3, 2, 8))])
def test_dwconv_nhwc_matches_fp32_conv(k, shape):
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(k)
    B, H, W, C = shape
    x = torch.randn(shape, device="cuda", generator=g).bfloat16()
    w = (torch.randn(C, 1, k, k, device="cuda", generator=g) / k).bfloat16()
    b = (torch.randn(C, device="cuda", generator=g) * 0.1).bfloat16()
    wt = w.reshape(C, k * k).t().contiguous()
    y = ops.dwconv_nhwc(x, wt, b, k)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=k // 2, groups=C).permute(0, 2, 3, 1)
    assert y.shape == x.shape and y.dtype == torch.bfloat16
    assert ((y.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-3 * ref.abs().max()).all()
    y0 = ops.dwconv_nhwc(x, wt, None, k)
    ref0 = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None, padding=k // 2, groups=C).permute(0, 2, 3, 1)
    assert ((y0.float() - ref0).abs() <= 2.0 ** -8 * ref0.abs() + 1e-3 * ref0.abs().max()).all()


def test_dwconv_rejects_bad_arguments():
    from visionllm_b200 import ops
    x = torch.zeros(1, 4, 4, 12, device="cuda", dtype=torch.bfloat16)           # C % 8 != 0
    with pytest.raises(RuntimeError):
        ops.dwconv_nhwc(x, torch.zeros(9, 12, device="cuda", dtype=torch.bfloat16), None, 3)
    x = torch.zeros(1, 4, 4, 16, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.dwconv_nhwc(x, torch.zeros(16, 16, device="cuda", dtype=torch.bfloat16), None, 4)   # even kernel


@pytest.mark.parametrize("cols", [64, 320, 2560])
def test_layernorm_gelu_matches_fp32(cols):
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cols)
    x = (torch.randn(37, cols, device="cuda", generator=g) * 2).bfloat16()
    w = (1 + 0.1 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    y = ops.layernorm(x, w, b, 1e-6, gelu=True)
    ref = F.gelu(F.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-6))
    assert ((y.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 2e-3).all()
    plain = ops.layernorm(x, w, b, 1e-6)
    assert ((plain.float() - F.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-6)).abs() <= 2.0 ** -7 * 4).all()


def test_internimage_matches_reference(golden_dir):
    from visionllm_b200.internimage import B200InternImage
    g = np.load(os.path.join(golden_dir, "mod_internimage_small.npz"))
    cfg = json.loads(str(g["cfg"]))
    m = B200InternImage(**cfg)
    assert json.loads(str(g["keys"])) == [list(k) for k in key_shapes(m)], "state-dict keys differ from the reference"
    m.load_state_dict(seeded_state_dict(m, 303))
    m = m.to("cuda", torch.bfloat16).eval()
    x = torch.from_numpy(g["pixel_values"]).cuda().bfloat16()
    outs = m(x)
    assert len(outs) == 4
    for i, o in enumerate(outs):
        assert getattr(o, "_b200_nhwc", False)
        ref32 = torch.from_numpy(g[f"out_f32_{i}"]).cuda().permute(0, 2, 3, 1)
        ref16 = torch.from_numpy(g[f"out_refbf16_{i}"]).cuda().permute(0, 2, 3, 1)
        assert o.shape == ref32.shape
        budget = 1.5 * rel_l2(ref16, ref32) + 1e-3
        assert rel_l2(o, ref32) <= budget, (i, rel_l2(o, ref32), budget)
    nchw = B200InternImage(channels_last_out=False, **cfg)
    nchw.load_state_dict(seeded_state_dict(nchw, 303))
    o2 = nchw.to("cuda", torch.bfloat16).eval()(x)
    assert all(torch.equal(a, b.permute(0, 3, 1, 2)) for a, b in zip(o2, outs))


@pytest.mark.parametrize("G,K,with_scale,pad", [(10, 9, True, 0), (2, 9, False, 2), (4, 25, True, 0)])
def test_dcnv3_prep_and_blend_match_torch(G, K, with_scale, pad):
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(G * K)
    cols = G * K * 3 + (G if with_scale else 0) + pad
    om = torch.randn(2, 5, 7, cols, device="cuda", generator=g) * 3
    off, mask, sc = ops.dcnv3_prep(om, G, K, with_scale)
    assert torch.equal(off, om[..., :G * K * 2])
    want = F.softmax(om[..., G * K * 2:G * K * 3].reshape(2, 5, 7, G, K), -1).reshape(2, 5, 7, G * K)
    assert (mask - want).abs().max().item() < 1e-6
    assert (mask.reshape(2, 5, 7, G, K).sum(-1) - 1).abs().max().item() < 1e-5
    if with_scale:
        assert (sc - om[..., G * K * 3:G * K * 3 + G].sigmoid()).abs().max().item() < 1e-6
    else:
        assert sc is None
    gc = 32
    core = torch.randn(2, 5, 7, G * gc, device="cuda", generator=g)
    xp = torch.randn(2, 5, 7, G * gc, device="cuda", generator=g)
    out = ops.dcnv3_blend(core, xp, sc, gc)
    if with_scale:
        s_ = sc[..., None].expand(2, 5, 7, G, gc).reshape(core.shape)
        ref = core * (1 - s_) + xp * s_
    else:
        ref = core
    assert out.dtype == torch.bfloat16 and torch.equal(out, ref.bfloat16()) or (out.float() - ref).abs().max() < 2e-2


def test_layernorm_residual_matches_fp32():
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(9)
    x = (torch.randn(3, 11, 640, device="cuda", generator=g) * 2).bfloat16()
    r = torch.randn(3, 11, 640, device="cuda", generator=g).bfloat16()
    w = (1 + 0.1 * torch.randn(640, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(640, device="cuda", generator=g)).bfloat16()
    y = ops.layernorm(x, w, b, 1e-6, residual=r)
    ref = r.float() + F.layer_norm(x.float(), (640,), w.float(), b.float(), 1e-6)
    assert ((y.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 2e-3).all()
