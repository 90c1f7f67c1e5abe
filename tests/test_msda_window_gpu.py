"""GPU: the TMA-staged window kernel of the encoder shape (csrc/msda_win.cu) against the C oracle and against the
global-memory warp-gather kernel it replaces.  The window only decides WHERE a corner row is read from (shared-memory
window filled by TMA or by cp.async vs global memory), never what is computed, so the two paths must agree BIT FOR BIT for any
window size -- including windows so small that most (query, head) pairs take the in-kernel fallback."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import msda_oracle as O  # noqa: E402
from visionllm_b200 import _lib  # noqa: E402


def enc_case(shapes_l, N, M, sigma, seed, outlier_frac=0.02, P=4, valid_ratio=None):
    """Encoder inputs: queries are the pixels, refs = pixel centres (optionally scaled by per-level valid ratios, as
    gd.py:1624-1646 does for padded images) + N(0, sigma) offsets; a fraction of samples is thrown anywhere in
    [-0.2, 1.2) (outside every window, partly outside the map)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = len(shapes_l)
    shapes = torch.tensor(shapes_l, dtype=torch.int64, device="cuda")
    lsi = torch.cat((shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]))
    S = int(shapes.prod(1).sum())
    refs = []
    for (H, W) in shapes_l:
        ys, xs = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32),
                                torch.arange(W, device="cuda", dtype=torch.float32), indexing="ij")
        refs.append(torch.stack(((xs + 0.5) / W, (ys + 0.5) / H), -1).reshape(-1, 2))
    ref = torch.cat(refs, 0)[None, :, None, None, None, :]
    if valid_ratio is not None:
        ref = ref * torch.tensor(valid_ratio, device="cuda", dtype=torch.float32).view(1, 1, 1, L, 1, 2)
    loc = ref + torch.randn(N, S, M, L, P, 2, device="cuda", generator=g) * sigma
    wild = torch.rand(N, S, M, L, P, 1, device="cuda", generator=g) < outlier_frac
    loc = torch.where(wild, torch.rand(N, S, M, L, P, 2, device="cuda", generator=g) * 1.4 - 0.2, loc).contiguous()
    value = torch.randn(N, S, M, 32, device="cuda", generator=g)
    attw = torch.softmax(torch.randn(N, S, M, L * P, device="cuda", generator=g), -1).view(N, S, M, L, P).contiguous()
    return value, shapes, lsi, loc, attw


def run(value, shapes, lsi, loc, attw, variant=_lib.MSDA_DEFAULT, window=(0, 0, 0), out_dtype=None, fill=-1):
    """value fp32 -> ms_deform_attn_forward; value bf16 -> ms_deform_attn_forward_bf16(out_dtype).  fill: the level mask of
    vllm_msda_set_window_fill; -1 leaves the library's default (every level by TMA), 0 = every level by cooperative cp.async."""
    import visionllm_b200.msda as ext
    if value.dtype == torch.float32 and variant == _lib.MSDA_DEFAULT:
        variant = _lib.MSDA_FP32_WINDOW                # fp32 rows: the window kernel is opt-in (the default is the patch kernel)
    with _lib.knob("msda_set_variant", variant), _lib.knob("msda_set_window", *window), \
            _lib.knob("msda_set_window_fill", fill):
        if value.dtype == torch.float32:
            return ext.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64)
        return ext.ms_deform_attn_forward_bf16(value, shapes, lsi, loc, attw, out_dtype)


def oracle(value, shapes, lsi, loc, attw):
    return torch.from_numpy(O.forward_kernel_semantics(value.float().cpu().numpy(), shapes.cpu().numpy(), lsi.cpu().numpy(),
                                                       loc.cpu().numpy(), attw.cpu().numpy())).cuda()


PYRAMIDS = {
    "pow2": [(32, 32), (16, 16), (8, 8), (4, 4)],
    "npot": [(25, 34), (13, 17), (7, 9), (4, 5)],                  # 800x1066-style non-power-of-two levels
    "wide": [(12, 50), (6, 25), (3, 13)],                          # 3 levels, K = 12
    "one": [(40, 40)],                                             # a single level
}


@pytest.mark.parametrize("pyr", list(PYRAMIDS))
@pytest.mark.parametrize("mode", ["f32", "bf16_f32out", "bf16_bf16out"])
def test_window_kernel_vs_oracle_and_bit_identical_to_global_path(pyr, mode):
    shapes_l = PYRAMIDS[pyr]
    value, shapes, lsi, loc, attw = enc_case(shapes_l, N=2, M=8, sigma=0.03, seed=11)
    if mode != "f32":
        value = value.bfloat16()
    od = {"f32": None, "bf16_f32out": torch.float32, "bf16_bf16out": torch.bfloat16}[mode]
    win = run(value, shapes, lsi, loc, attw, out_dtype=od)
    glob = run(value, shapes, lsi, loc, attw, variant=_lib.MSDA_BF16_NO_WINDOW if mode != "f32" else _lib.MSDA_NO_HINT,
               out_dtype=od)
    assert torch.equal(win, glob), (win.float() - glob.float()).abs().max().item()
    # the two window-fill mechanisms (one TMA box per level, the default; cooperative cp.async) give the same bits
    assert torch.equal(run(value, shapes, lsi, loc, attw, out_dtype=od, fill=0), win)
    ref = oracle(value, shapes, lsi, loc, attw)
    scale = ref.abs().max().item()
    if win.dtype == torch.float32:
        assert (win - ref).abs().max().item() <= 1e-5 * max(1.0, scale)
    else:
        assert ((win.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-5 * scale).all()


@pytest.mark.parametrize("window", [(8, 16, 1), (4, 4, 2), (16, 16, 12), (8, 8, 3), (2, 3, 1)])
def test_result_does_not_depend_on_the_window_geometry(window):
    """Tiny windows push most pairs through the in-kernel global fallback, large ones none: same bits every time."""
    value, shapes, lsi, loc, attw = enc_case(PYRAMIDS["npot"], N=1, M=8, sigma=0.04, seed=3, outlier_frac=0.05)
    base32 = run(value, shapes, lsi, loc, attw, variant=_lib.MSDA_NO_HINT)
    base16 = run(value.bfloat16(), shapes, lsi, loc, attw, variant=_lib.MSDA_BF16_NO_WINDOW, out_dtype=torch.float32)
    assert torch.equal(run(value, shapes, lsi, loc, attw, window=window), base32)
    assert torch.equal(run(value.bfloat16(), shapes, lsi, loc, attw, window=window, out_dtype=torch.float32), base16)


def test_padded_image_valid_ratios_and_pixel_centre_references():
    """Reference points exactly on pixel centres (sigma = 0: the adversarial floor() case of SURVEY App. A) and scaled
    by per-level valid ratios as for a padded batch entry."""
    vr = [(0.8, 0.75), (0.8235, 0.7692), (0.7778, 0.8571), (0.8, 0.75)]
    for sigma, ratio in ((0.0, None), (0.0, vr), (0.02, vr)):
        value, shapes, lsi, loc, attw = enc_case(PYRAMIDS["npot"], N=1, M=8, sigma=sigma, seed=5, outlier_frac=0.0,
                                                 valid_ratio=ratio)
        win = run(value, shapes, lsi, loc, attw)
        ref = oracle(value, shapes, lsi, loc, attw)
        assert (win - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())
        assert torch.equal(win, run(value, shapes, lsi, loc, attw, variant=_lib.MSDA_NO_HINT))


def test_out_of_range_samples_and_unsampled_nans_do_not_leak():
    """(a) every sample out of range, value all NaN -> exact zeros (weight 0 never meets a NaN: the zero row);
    (b) NaNs in pixels no sample touches (but which the TMA does load into the windows) stay invisible."""
    shapes_l = PYRAMIDS["pow2"]
    value, shapes, lsi, loc, attw = enc_case(shapes_l, N=1, M=8, sigma=0.0, seed=1, outlier_frac=0.0)
    nan_value = torch.full_like(value, float("nan"))
    far = (loc * 0 + 7.0).contiguous()
    for v in (nan_value, nan_value.bfloat16()):
        out = run(v, shapes, lsi, far, attw, out_dtype=torch.float32)
        assert (out == 0).all()
    # samples confined to the top-left 2x2 pixels of every level; NaN everywhere else in the maps
    S = value.shape[1]
    keep = torch.zeros(S, dtype=torch.bool, device="cuda")
    for (H, W), s0 in zip(shapes_l, lsi.tolist()):
        for y in range(3):
            keep[s0 + y * W: s0 + y * W + 3] = True
    v = value.clone()
    v[:, ~keep] = float("nan")
    near = torch.rand_like(loc)
    for l, (H, W) in enumerate(shapes_l):
        near[:, :, :, l, :, 0] = (0.6 + 1.3 * near[:, :, :, l, :, 0]) / W     # w_im in [0.1, 1.4): corners in columns 0..2
        near[:, :, :, l, :, 1] = (0.6 + 1.3 * near[:, :, :, l, :, 1]) / H
    near = near.contiguous()
    out = run(v, shapes, lsi, near, attw)
    ref = oracle(value, shapes, lsi, near, attw)
    assert torch.isfinite(out).all() and (out - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())


def test_full_size_encoder_shape_properties():
    """BASELINE cfg 2b encoder shape (S = 21760): window == global path bit for bit, partition of unity, linearity."""
    import bench_workloads as B
    value, shapes, lsi, loc, attw = B.msda_encoder_inputs(torch, 2, torch.device("cuda"), 77)
    hs = shapes.cpu()
    import visionllm_b200.msda as ext
    win = run(value, shapes, lsi, loc, attw)
    assert torch.equal(win, run(value, shapes, lsi, loc, attw, variant=_lib.MSDA_NO_HINT))
    assert torch.equal(win, ext.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64, host_shapes=hs))   # default path
    strict = ext.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64, flags=ext.STRICT)
    assert (win - strict).abs().max().item() <= 1e-5 * strict.abs().max().item()
    v16 = value.bfloat16()
    w16 = ext.ms_deform_attn_forward_bf16(v16, shapes, lsi, loc, attw, torch.float32)
    assert torch.equal(w16, run(v16, shapes, lsi, loc, attw, variant=_lib.MSDA_BF16_NO_WINDOW, out_dtype=torch.float32))
    assert (w16 - ext.ms_deform_attn_forward(v16.float(), shapes, lsi, loc, attw, 64, flags=ext.STRICT)).abs().max().item() \
        <= 1e-5 * strict.abs().max().item()
    ones = torch.ones_like(value)
    inner = loc.clamp(0.1, 0.9).contiguous()
    assert (ext.ms_deform_attn_forward(ones, shapes, lsi, inner, attw, 64) - 1.0).abs().max().item() < 1e-5


@pytest.mark.parametrize("pyr", ["pow2", "npot"])
def test_fused_module_input_is_bit_identical_to_the_torch_glue(pyr):
    """GroundingDinoMultiscaleDeformableAttention (encoder self-attention, bf16): softmax over the 16 logits, offset /
    (W, H) in bf16 and reference + offset in fp32 computed INSIDE the gather kernel must reproduce the five torch
    elementwise kernels of the unfused path bit for bit -- output and returned attention weights."""
    from types import SimpleNamespace
    import visionllm_b200.msda as msda_ext
    from visionllm_b200.gdino import GroundingDinoMultiscaleDeformableAttention
    shapes_l = PYRAMIDS[pyr]
    cfg = SimpleNamespace(d_model=256, num_feature_levels=4, disable_custom_kernels=False)
    torch.manual_seed(0)
    m = GroundingDinoMultiscaleDeformableAttention(cfg, num_heads=8, n_points=4)
    with torch.no_grad():
        m.attention_weights.weight.normal_(0, 0.05); m.attention_weights.bias.normal_(0, 0.5)
        m.sampling_offsets.weight.normal_(0, 0.02)
    m = m.to("cuda", torch.bfloat16).eval()
    shapes = torch.tensor(shapes_l, dtype=torch.int64, device="cuda")
    msda_ext.attach_host_shapes(shapes, shapes_l)
    lsi = torch.cat((shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]))
    S = int(shapes.prod(1).sum())
    B = 2
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, S, 256, device="cuda", generator=g).bfloat16()
    pos = (torch.randn(B, S, 256, device="cuda", generator=g) * 0.3).bfloat16()
    refs = []
    for (H, W) in shapes_l:
        ys, xs = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32),
                                torch.arange(W, device="cuda", dtype=torch.float32), indexing="ij")
        refs.append(torch.stack(((xs + 0.5) / W, (ys + 0.5) / H), -1).reshape(-1, 2))
    ref = torch.cat(refs, 0)[None, :, None, :].repeat(B, 1, 4, 1) * torch.tensor([[0.9, 0.8]], device="cuda").view(1, 1, 1, 2)
    mask = torch.ones(B, S, dtype=torch.bool, device="cuda")
    mask[1, -7:] = False
    kw = dict(hidden_states=x, attention_mask=mask, encoder_hidden_states=x, position_embeddings=pos,
              reference_points=ref.contiguous(), spatial_shapes=shapes, level_start_index=lsi)
    a_out, a_w = m(**kw)
    msda_ext.FUSED_MODULE_INPUT = False
    try:
        b_out, b_w = m(**kw)
    finally:
        msda_ext.FUSED_MODULE_INPUT = True
    assert a_w.dtype == torch.bfloat16 and a_w.shape == b_w.shape == (B, S, 8, 4, 4)
    assert torch.equal(a_w, b_w)
    assert torch.equal(a_out, b_out), (a_out.float() - b_out.float()).abs().max().item()
