"""GPU: visionllm_b200.swin.B200SwinBackbone (our GEMM / LayerNorm / window-attention kernels) against HF's
`SwinBackbone` -- the third-party module the reference instantiates (modeling_ov_grounding_dino_mask_dn.py:483) --
run by torch on the same GPU: fp32 as the oracle, bf16 as "the reference's deployed precision".
Tolerance: rel_l2(ours, hf_fp32) <= 1.5 * rel_l2(hf_bf16, hf_fp32) + 1e-3 per feature map."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize("hw,ws,embed,heads,depths", [
    ((224, 288), 7, 96, [3, 6, 12, 24], [2, 2, 2, 2]),        # Swin-T widths, divisible by the window
    ((200, 264), 7, 96, [3, 6, 12, 24], [2, 2, 2, 2]),        # 50x66 tokens: padded to 56x70, odd merges later
    ((96, 128), 4, 32, [1, 2, 4, 8], [2, 2, 2, 2]),           # the whole-stage test's backbone
    ((192, 192), 12, 64, [2, 4, 8, 16], [2, 2, 2, 2]),        # window 12 (Swin-B/L style), 144-token windows
])
def test_swin_backbone_vs_hf_on_gpu(hw, ws, embed, heads, depths):
    from transformers import SwinConfig
    from transformers.models.swin.modeling_swin import SwinBackbone
    from weights_util import seeded_state_dict
    from visionllm_b200.swin import B200SwinBackbone
    cfg = SwinConfig(image_size=224, embed_dim=embed, depths=depths, num_heads=heads, window_size=ws,
                     out_features=["stage1", "stage2", "stage3", "stage4"])
    hf = SwinBackbone(cfg).eval()
    sd = seeded_state_dict(hf, 17)
    hf.load_state_dict(sd)
    ours = B200SwinBackbone(cfg).eval()
    ours.load_state_dict(sd, strict=True)
    ours = ours.cuda().bfloat16()
    x = torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(2)).bfloat16()
    with torch.no_grad():
        hf = hf.cuda()
        f32 = hf(x.cuda().float()).feature_maps
        f16 = hf.bfloat16()(x.cuda()).feature_maps
        mine = ours(x.cuda()).feature_maps
    for i, (a, b, c) in enumerate(zip(f32, f16, mine)):
        c = c.permute(0, 3, 1, 2)
        assert c.shape == a.shape
        e_ref, e = rel(b, a), rel(c, a)
        assert e <= 1.5 * e_ref + 1e-3, f"stage{i + 1}: ours {e:.5f} vs hf-bf16 {e_ref:.5f}"


@pytest.mark.parametrize("T,H,D,nB", [(49, 3, 32, 4), (144, 2, 32, 1), (16, 8, 32, 6), (49, 2, 64, 3), (64, 5, 32, 2), (1, 2, 32, 1)])
def test_attention_additive_bias(T, H, D, nB):
    """attn_bias [nB, H, T, T] fp32, batch b uses slab b % nB (incl. -100 shift-mask entries)."""
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(T)
    B = nB * 3
    q, k, v = (torch.randn(B, T, H, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    bias = torch.randn(nB, H, T, T, device="cuda", generator=g)
    bias[torch.rand(nB, 1, T, T, device="cuda", generator=g).expand(-1, H, -1, -1) < 0.2] += -100.0
    out = ops.attention(q, k, v, attn_bias=bias.contiguous())
    s = (q.float().permute(0, 2, 1, 3) @ k.float().permute(0, 2, 3, 1)) * D ** -0.5 + bias.repeat(3, 1, 1, 1)
    ref = (torch.softmax(s, -1) @ v.float().permute(0, 2, 1, 3)).permute(0, 2, 1, 3).reshape(B, T, H * D)
    assert rel(out, ref) < 6e-3
    if D == 32 and T <= 64:
        # r2: these calls take the one-warp-per-(window, head) kernel; same arithmetic order as the general kernel
        from visionllm_b200 import _lib
        with _lib.knob("attention_set_variant", _lib.ATTN_WARP_MMA):
            general = ops.attention(q, k, v, attn_bias=bias.contiguous())
        assert torch.equal(out, general)
        qkv = torch.randn(B, T, 3, H, D, device="cuda", generator=g).bfloat16()          # packed, strided views like swin.py
        o1 = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], attn_bias=bias.contiguous())
        with _lib.knob("attention_set_variant", _lib.ATTN_WARP_MMA):
            o2 = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], attn_bias=bias.contiguous())
        assert torch.equal(o1, o2)
    with pytest.raises(RuntimeError):
        ops.attention(q, k, v, attn_bias=bias[:, :, :, :-1].contiguous())


def test_layernorm_gather_kernel_equals_layernorm_then_gather():
    """ops.layernorm_gather (LN + zero pad + row gather of the Swin window partition in one pass) must be bit-identical to
    ops.layernorm followed by cat(zero row) + index_select -- rows are independent, the arithmetic is the same kernel's."""
    from visionllm_b200 import ops
    from visionllm_b200.swin import _window_rows
    g = torch.Generator(device="cuda").manual_seed(4)
    for (H, W, ws, shift, C) in ((10, 13, 7, 3, 96), (16, 16, 4, 0, 192), (9, 9, 7, 3, 48)):
        B = 3
        x = torch.randn(B, H * W, C, device="cuda", generator=g).bfloat16()
        w = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
        b = (0.1 * torch.randn(C, device="cuda", generator=g)).bfloat16()
        fwd, inv, Hp, Wp = _window_rows(H, W, ws, shift, x.device)
        got = ops.layernorm_gather(x, fwd, w, b, 1e-5)
        h = ops.layernorm(x, w, b, 1e-5)
        h = torch.cat((h, h.new_zeros(B, 1, C)), 1)
        assert torch.equal(got, h.index_select(1, fwd))
        assert torch.equal(got.index_select(1, inv), ops.layernorm(x, w, b, 1e-5))      # the inverse map drops the pads
