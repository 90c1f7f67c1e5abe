"""GPU: region-encoder training (visionllm_b200/train.py region_encoder_train, csrc/train_ops.cu) -- the LayerNorm -> GELU
backward and the point-pool backward against float64, the module's gradients against the reference's own RegionEncoder
(tests/golden/train_region_encoder.npz) and the composite step with regions.

Checkers are those of tests/bf16_rounding.py (`rounds` / `within`, no max|ref| term).  Bounds, u = 2^-24:
  LN -> GELU dx   statistics as the forward's (ln_stats): with d = 8 VPT + 13, rstd is within er = (d / 2 + 6) u
                  relatively and n = (x - mean) rstd within en = |n| er + rstd d u mean|x|; z = n w + b within
                  ez = |w| en + 2u (|z| + |w n|); g = dy gelu'(z) within eg = |dy| (|gelu''(z)| ez + 16u (Phi(z) +
                  |z| phi(z) (1 + z^2)) + 4u) (the GELU backward's bound); dx = rstd (w g - m1 - n m2) within
                  |dx| er + rstd (|w| eg + mean|w| eg + |n| mean(|w| (|n| eg + |g| en)) + en |m2|
                  + (d + 4) u (|w g| + mean|w g| + |n| mean|w g n|)).
  LN dw / db      sums over rows of g n and g: sum(|n| eg + |g| en) (+ eg) + c u sum|g n| (sum|g|), c = rows per slot +
                  ceil(slots / 8) + 10 (the slot's chain, the 8-warp partial chain and tree).
  point pool      a_l = sum over points of pw * corner weight (fp32 chain over the n points of the level, the corner weight
                  two fp32 roundings, 1 - lh one): |a_l - a_l64| <= (n + 4) u A_l, A_l = sum |pw cw|; the output
                  sum_l a_l g_l / c_l within sum_l |g_l| / c_l (A_l (n + 4) u + 2u A_l) + L u sum_l |a_l g_l / c_l|.
  modules         rel_l2(ours, fp32 ref) <= 2 rel_l2(bf16 ref, fp32 ref) + 3e-3 (the module rule of the chat step).
"""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bf16_rounding import U, note_ratio, print_report, rounds, within
from test_train_kernels_contract_gpu import EALIGN, EINVAL, NAN, bits, gen, same_bits
from visionllm_b200 import _lib

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from weights_util import key_shapes, seeded_state_dict  # noqa: E402

EUNSUPPORTED = -2


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print_report("region encoder training")


def stream():
    return torch.cuda.current_stream().cuda_stream


def rel(a, b):
    return float(torch.linalg.norm((a.double() - b.double()).flatten()) / (torch.linalg.norm(b.double().flatten()) + 1e-300))


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm -> GELU backward
# ---------------------------------------------------------------------------------------------------------------------
def ln_gelu_call(x, w, b, dy, dx, dw, db, part, n_part, rows, cols, eps=1e-6):
    return _lib.lib().vllm_layernorm_gelu_bwd_bf16(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), dy.data_ptr(),
                                                   dy.stride(0), dx.data_ptr(), dx.stride(0), dw.data_ptr(), db.data_ptr(),
                                                   part.data_ptr(), n_part, rows, cols, eps, stream())


def ln_gelu_vpt(cols):
    nvec = cols // 8
    if nvec <= 128:
        return 1 if nvec <= 32 else (2 if nvec <= 64 else 4)
    if nvec <= 1024:
        return 2 if nvec <= 256 else (4 if nvec <= 512 else 8)
    return 8


def ln_gelu_run(x, w, b, dy, eps=1e-6, ld=None):
    rows, cols = x.shape
    ld = ld or cols
    n_part = _lib.lib().vllm_layernorm_gelu_bwd_partials(rows)
    part = torch.empty((2 * max(n_part, 1), cols), dtype=torch.float32, device="cuda")
    buf = torch.full((rows, ld), NAN, dtype=torch.bfloat16, device="cuda")
    dx = buf[:, :cols]
    dw = torch.full((cols,), NAN, device="cuda")
    db = torch.full((cols,), NAN, device="cuda")
    assert ln_gelu_call(x, w, b, dy, dx, dw, db, part, n_part, rows, cols, eps) == 0
    torch.cuda.synchronize()
    if ld > cols:
        assert buf[:, cols:].isnan().all()
    return dx, dw, db, n_part


def ln_gelu_ref(x, w, b, dy, eps, cols, rows, n_part):
    """float64 reference and the bounds of the module docstring."""
    x, w, b, dy = (t.double() for t in (x, w, b, dy))
    mean = x.mean(1, keepdim=True)
    rstd = ((x - mean).pow(2).mean(1, keepdim=True) + eps).rsqrt()
    n = (x - mean) * rstd
    z = n * w + b
    Phi = 0.5 * (1 + torch.erf(z / math.sqrt(2)))
    phi = torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    gp = Phi + z * phi
    gpp = phi * (2 - z * z)
    g = dy * gp
    wg = w * g
    m1 = wg.mean(1, keepdim=True)
    m2 = (wg * n).mean(1, keepdim=True)
    dx = rstd * (wg - m1 - n * m2)
    d = 8 * ln_gelu_vpt(cols) + 13
    er = (d / 2 + 6) * U
    en = n.abs() * er + rstd * d * U * x.abs().mean(1, keepdim=True)
    ez = w.abs() * en + 2 * U * (z.abs() + (w * n).abs())
    eg = dy.abs() * (gpp.abs() * ez + 16 * U * (Phi + z.abs() * phi * (1 + z * z)) + 4 * U)
    Edx = (dx.abs() * er + rstd * (w.abs() * eg + (w.abs() * eg).mean(1, keepdim=True)
                                   + n.abs() * (w.abs() * (n.abs() * eg + g.abs() * en)).mean(1, keepdim=True)
                                   + en * m2.abs()
                                   + (d + 4) * U * (wg.abs() + wg.abs().mean(1, keepdim=True)
                                                    + n.abs() * (wg * n).abs().mean(1, keepdim=True))))
    rps = -(-rows // max(n_part, 1))
    c = rps + -(-n_part // 8) + 10
    dw = (g * n).sum(0)
    db = g.sum(0)
    Edw = (n.abs() * eg + g.abs() * en).sum(0) + c * U * (g * n).abs().sum(0)
    Edb = eg.sum(0) + c * U * g.abs().sum(0)
    return dx, dw, db, Edx, Edw, Edb


def ln_gelu_inputs(rows, cols, g):
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 1.5 + 0.3).bfloat16()
    w = (1 + 0.3 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    b = (0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    dy = torch.randn(rows, cols, device="cuda", generator=g).bfloat16()
    return x, w, b, dy


@pytest.mark.parametrize("cols", [16, 64, 72, 256, 1024, 3200])
@pytest.mark.parametrize("rows", [1, 37, 4099])
def test_layernorm_gelu_backward_vs_fp64(cols, rows):
    g = gen(cols * 7 + rows)
    x, w, b, dy = ln_gelu_inputs(rows, cols, g)
    ld = cols + 24
    xb = torch.full((rows, ld), NAN, dtype=torch.bfloat16, device="cuda")
    xb[:, :cols] = x
    dyb = torch.full((rows, ld + 8), NAN, dtype=torch.bfloat16, device="cuda")
    dyb[:, :cols] = dy
    dx, dw, db, n_part = ln_gelu_run(xb[:, :cols], w, b, dyb[:, :cols], ld=ld + 16)
    rdx, rdw, rdb, Edx, Edw, Edb = ln_gelu_ref(x, w, b, dy, 1e-6, cols, rows, n_part)
    rounds(dx, rdx, Edx, "ln_gelu_bwd_dx", f"{rows}x{cols}")
    within(dw, rdw, Edw, "ln_gelu_bwd_dw", f"{rows}x{cols}")
    within(db, rdb, Edb, "ln_gelu_bwd_db", f"{rows}x{cols}")
    again = ln_gelu_run(xb[:, :cols], w, b, dyb[:, :cols], ld=ld + 16)
    assert all(same_bits(a, b_) for a, b_ in zip((dx.contiguous(), dw, db), (again[0].contiguous(), again[1], again[2])))


def test_layernorm_gelu_backward_exact_probes():
    g = gen(5)
    for cols in (64, 256, 3200):
        x, w, b, dy = ln_gelu_inputs(300, cols, g)
        dx, dw, db, _ = ln_gelu_run(x, w, b, torch.zeros_like(dy))
        assert (dx == 0).all() and (dw == 0).all() and (db == 0).all(), cols
        dx, _, _, _ = ln_gelu_run(x, torch.zeros_like(w), b, dy)
        assert (dx == 0).all(), cols


def test_layernorm_gelu_backward_rejections_leave_outputs_untouched():
    g = gen(6)
    rows, cols = 100, 64
    x, w, b, dy = ln_gelu_inputs(rows, cols, g)
    n_part = _lib.lib().vllm_layernorm_gelu_bwd_partials(rows)
    part = torch.full((2 * n_part, cols), NAN, device="cuda")
    dx = torch.full((rows, cols), NAN, dtype=torch.bfloat16, device="cuda")
    dw = torch.full((cols,), NAN, device="cuda")
    db = torch.full((cols,), NAN, device="cuda")
    before = [bits(t).clone() for t in (dx, dw, db, part)]
    odd = torch.zeros(rows, cols + 8, dtype=torch.bfloat16, device="cuda")
    L = _lib.lib()
    cases = [
        (ln_gelu_call(x, w, b, dy, dx, dw, db, part, n_part - 1, rows, cols), EINVAL),             # too few partials
        (ln_gelu_call(x, w, b, dy, dx, dw, db, part, n_part, -1, cols), EINVAL),
        (L.vllm_layernorm_gelu_bwd_bf16(x.data_ptr(), cols, w.data_ptr(), b.data_ptr(), dy.data_ptr(), cols, dx.data_ptr(),
                                        cols, dw.data_ptr(), db.data_ptr(), part.data_ptr(), n_part, rows, 60, 1e-6,
                                        stream()), EUNSUPPORTED),                                        # cols % 8
        (L.vllm_layernorm_gelu_bwd_bf16(x.data_ptr(), cols, w.data_ptr(), b.data_ptr(), dy.data_ptr(), cols, dx.data_ptr(),
                                        cols, dw.data_ptr(), db.data_ptr(), part.data_ptr(), n_part, rows, 16392, 1e-6,
                                        stream()), EUNSUPPORTED),                                        # wider than the forward
        (L.vllm_layernorm_gelu_bwd_bf16(odd[:, 1:].data_ptr(), cols + 8, w.data_ptr(), b.data_ptr(), dy.data_ptr(), cols,
                                        dx.data_ptr(), cols, dw.data_ptr(), db.data_ptr(), part.data_ptr(), n_part, rows,
                                        cols, 1e-6, stream()), EALIGN),
        (L.vllm_layernorm_gelu_bwd_bf16(x.data_ptr(), 68, w.data_ptr(), b.data_ptr(), dy.data_ptr(), cols, dx.data_ptr(),
                                        cols, dw.data_ptr(), db.data_ptr(), part.data_ptr(), n_part, rows, cols, 1e-6,
                                        stream()), EALIGN),                                              # pitch % 8
        (L.vllm_layernorm_gelu_bwd_bf16(x.data_ptr(), cols, w.data_ptr(), None, dy.data_ptr(), cols, dx.data_ptr(), cols,
                                        dw.data_ptr(), db.data_ptr(), part.data_ptr(), n_part, rows, cols, 1e-6,
                                        stream()), EINVAL),
    ]
    torch.cuda.synchronize()
    for i, (rc, want) in enumerate(cases):
        assert rc == want, (i, rc, want)
    assert all(torch.equal(bits(t), b_) for t, b_ in zip((dx, dw, db, part), before))


# ---------------------------------------------------------------------------------------------------------------------
# point-pool backward
# ---------------------------------------------------------------------------------------------------------------------
def pool_call(loc, wgt, cnt, grad, h, w, density, out):
    levels, R, n = wgt.shape
    return _lib.lib().vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), levels, R,
                                               h, w, grad.shape[-1], density.data_ptr(), out.data_ptr(), stream())


def pool_run(loc, wgt, grad, h, w):
    levels, R, n = wgt.shape
    cnt = wgt.sum(2).contiguous()
    out = torch.full((R, h * w, grad.shape[-1]), NAN, dtype=torch.bfloat16, device="cuda")
    dens = torch.empty((levels, R, h * w), device="cuda")
    assert pool_call(loc, wgt, cnt, grad, h, w, dens, out) == 0
    torch.cuda.synchronize()
    return out


def corner_matrix(loc, wgt, h, w):
    """fp64 [levels, R, h*w] matrices S (pw * corner weight, summed over points) and A (|.|), with the kernel's fp32 corner
    geometry (loc * size - 0.5 and the fractional parts in fp32; corners outside the map dropped)."""
    levels, R, n = wgt.shape
    x, y = loc[..., 0].float(), loc[..., 1].float()
    h_im = y * h - 0.5                                            # two fp32 roundings, as msda_geom
    w_im = x * w - 0.5
    inside = (h_im > -1) & (w_im > -1) & (h_im < h) & (w_im < w)
    hl, wl = torch.floor(h_im), torch.floor(w_im)
    lh, lw = (h_im - hl).double(), (w_im - wl).double()
    S = torch.zeros(levels, R, h * w, dtype=torch.float64, device="cuda")
    A = torch.zeros_like(S)
    pw = wgt.double() * inside
    for dh, dw_, cw in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
        py, px = hl.long() + dh, wl.long() + dw_
        ok = inside & (py >= 0) & (py < h) & (px >= 0) & (px < w)
        idx = (py * w + px).clamp(0, h * w - 1)
        v = torch.where(ok, pw * cw, torch.zeros_like(cw))
        S.scatter_add_(2, idx, v)
        A.scatter_add_(2, idx, v.abs())
    return S, A


def pool_ref(loc, wgt, grad, h, w):
    S, A = corner_matrix(loc, wgt, h, w)
    levels, R, n = wgt.shape
    cnt = wgt.double().sum(2)
    t = torch.where(cnt[..., None] > 0, grad.double() / cnt.clamp(min=1)[..., None], torch.zeros_like(grad.double()))
    ref = torch.einsum("lrp,lrc->rpc", S, t)
    E = (torch.einsum("lrp,lrc->rpc", A, t.abs()) * (n + 6) * U + levels * U * torch.einsum("lrp,lrc->rpc", S.abs(), t.abs()))
    return ref, E, S


def pool_inputs(levels, R, n_list, g):
    n = max(max(n_list), 1)
    n = (n + 15) // 16 * 16
    loc = torch.zeros(levels, R, n, 2, device="cuda")
    wgt = torch.zeros(levels, R, n, device="cuda")
    for lv in range(levels):
        for r, k in enumerate(n_list):
            if k:
                loc[lv, r, :k] = torch.rand(k, 2, device="cuda", generator=g)
                wgt[lv, r, :k] = 1
    return loc, wgt


@pytest.mark.parametrize("h,w,C", [(8, 8, 256), (32, 32, 64), (5, 7, 40)])
def test_point_pool_backward_vs_fp64(h, w, C):
    g = gen(h * w + C)
    n_list = [2304, 9, 0, 700]
    loc, wgt = pool_inputs(3, 4, n_list, g)
    grad = torch.randn(3, 4, C, device="cuda", generator=g).bfloat16()
    out = pool_run(loc, wgt, grad, h, w)
    ref, E, S = pool_ref(loc, wgt, grad, h, w)
    rounds(out, ref, E, "point_pool_bwd", f"{h}x{w}x{C}")
    assert (out[2] == 0).all()                                   # the empty region
    assert same_bits(out, pool_run(loc, wgt, grad, h, w))        # run-to-run identical
    # adjoint identity in fp64: <pool(E), g> == <E, pool^T(g)> with the forward restated as bilinear grid_sample
    emb = torch.randn(4, h, w, C, device="cuda", generator=g, dtype=torch.float64)
    grid = (loc.double() * 2 - 1).view(3 * 4, -1, 1, 2)
    samp = F.grid_sample(emb.permute(0, 3, 1, 2).repeat(3, 1, 1, 1), grid, align_corners=False).squeeze(-1)   # [3*4, C, n]
    cnt = wgt.double().sum(2).view(-1)
    pooled = ((samp * wgt.double().view(12, 1, -1)).sum(-1) / cnt[:, None]).nan_to_num().view(3, 4, C)
    lhs = float((pooled * grad.double()).sum())
    rhs = float((emb.reshape(4, h * w, C) * out.double()).sum())
    scale = float((emb.abs().reshape(4, h * w, C) * (ref.abs() + E)).sum())
    assert abs(lhs - rhs) <= 2 * float((emb.abs().reshape(4, h * w, C) * E).sum()) + 1e-5 * scale + 0.01 * scale * 2 ** -8, \
        (lhs, rhs)


def test_point_pool_backward_exact_probes():
    h, w, C = 4, 8, 16
    g = gen(9)
    grad = (2.0 ** torch.randint(-3, 3, (2, 3, C), device="cuda", generator=g).float()).bfloat16()
    # points at pixel centres ((j + 0.5) / size is exact in fp32 here), power-of-two g and counts: every output exact.
    # Region 0: four points (one pixel twice) on level 0 only; region 1: two points on both levels; region 2: empty.
    loc = torch.zeros(2, 3, 16, 2, device="cuda")
    wgt = torch.zeros(2, 3, 16, device="cuda")
    for k, (py, px) in enumerate(((0, 0), (1, 3), (3, 7), (1, 3))):
        loc[0, 0, k] = torch.tensor([(px + 0.5) / w, (py + 0.5) / h])
        wgt[0, 0, k] = 1
    loc[:, 1, :2] = torch.tensor([[0.5 / w, 0.5 / h], [2.5 / w, 1.5 / h]])
    wgt[:, 1, :2] = 1
    out = pool_run(loc, wgt, grad, h, w).double()
    want = torch.zeros(3, h * w, C, dtype=torch.float64, device="cuda")
    for py, px, k in ((0, 0, 1), (1, 3, 2), (3, 7, 1)):
        want[0, py * w + px] = k * grad[0, 0].double() / 4
    for py, px in ((0, 0), (1, 2)):
        want[1, py * w + px] = grad[0, 1].double() / 2 + grad[1, 1].double() / 2
    assert torch.equal(out, want)
    # border points (0, 0) and (1 - ulp, 1 - ulp): each keeps one corner inside the map, of weight 1/4 (the second one
    # 1/4 (1 + 3 * 2^-22) in fp32, which rounds to 1/4 in bf16 after g / 2); every other pixel exact 0
    one_m = float(np.nextafter(np.float32(1), np.float32(0)))
    loc = torch.zeros(1, 1, 16, 2, device="cuda")
    wgt = torch.zeros(1, 1, 16, device="cuda")
    loc[0, 0, 1] = torch.tensor([one_m, one_m])
    wgt[0, 0, :2] = 1
    out = pool_run(loc, wgt, grad[:1, :1].contiguous(), h, w).double()
    want = torch.zeros(1, h * w, C, dtype=torch.float64, device="cuda")
    want[0, 0] = want[0, h * w - 1] = grad[0, 0].double() / 8
    assert torch.equal(out, want)


def test_point_pool_backward_rejections_leave_outputs_untouched():
    loc, wgt = pool_inputs(2, 2, [20, 3], gen(3))
    grad = torch.randn(2, 2, 32, device="cuda").bfloat16()
    cnt = wgt.sum(2).contiguous()
    out = torch.full((2, 16, 32), NAN, dtype=torch.bfloat16, device="cuda")
    dens = torch.full((2, 2, 16), NAN, device="cuda")
    before = [bits(out).clone(), bits(dens).clone()]
    L = _lib.lib()
    n = wgt.shape[2]
    odd = torch.zeros(2 * 2 * 32 + 8, dtype=torch.bfloat16, device="cuda")
    cases = [
        (L.vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), 0, 2, 4, 4, 32,
                                    dens.data_ptr(), out.data_ptr(), stream()), EINVAL),
        (L.vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), 2, 2, 0, 4, 32,
                                    dens.data_ptr(), out.data_ptr(), stream()), EINVAL),
        (L.vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), 2, 2, 4, 4, 36,
                                    dens.data_ptr(), out.data_ptr(), stream()), EUNSUPPORTED),
        (L.vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, odd[1:].data_ptr(), 2, 2, 4, 4, 32,
                                    dens.data_ptr(), out.data_ptr(), stream()), EALIGN),
        (L.vllm_point_pool_bwd_bf16(None, wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), 2, 2, 4, 4, 32,
                                    dens.data_ptr(), out.data_ptr(), stream()), EINVAL),
    ]
    torch.cuda.synchronize()
    for i, (rc, want) in enumerate(cases):
        assert rc == want, (i, rc, want)
    assert torch.equal(bits(out), before[0]) and torch.equal(bits(dens), before[1])


# ---------------------------------------------------------------------------------------------------------------------
# the module against the reference's own RegionEncoder
# ---------------------------------------------------------------------------------------------------------------------
def golden_module(golden_dir):
    from visionllm_b200.region_encoder import B200RegionEncoder
    gz = np.load(os.path.join(golden_dir, "train_region_encoder.npz"))
    cfg = json.loads(str(gz["cfg"]))
    m = B200RegionEncoder(mask_pool_type="grid_sample", **cfg)
    assert json.loads(str(gz["keys"])) == [list(k) for k in key_shapes(m)]
    m.load_state_dict(seeded_state_dict(m, 77))
    m = m.to("cuda", torch.bfloat16)
    B = gz["images"].shape[0]
    feats = [torch.from_numpy(gz[f"feat_{i}"]).cuda().bfloat16() for i in range(3)]
    pts = [[torch.from_numpy(gz[f"points_{lv}_{i}"]).cuda() for i in range(B)] for lv in range(3)]
    images = torch.from_numpy(gz["images"]).cuda().bfloat16()
    masks = torch.from_numpy(gz["masks"]).cuda().bfloat16()
    return gz, m, images, masks, feats, pts


def test_region_encoder_gradients_match_reference(golden_dir):
    from visionllm_b200.train import region_encoder_train
    gz, m, images, masks, feats, pts = golden_module(golden_dir)
    out = region_encoder_train(m, images, masks, feats, sample_points=pts)
    out.backward(torch.from_numpy(gz["grad_out"]).cuda().bfloat16())
    for n in json.loads(str(gz["params"])):
        p = dict(m.named_parameters())[n]
        r32 = torch.from_numpy(gz[f"grad_f32/{n}"]).cuda()
        r16 = torch.from_numpy(gz[f"grad_refbf16/{n}"]).cuda()
        assert p.grad is not None and p.grad.shape == r32.shape, n
        a, b = rel(p.grad, r32), rel(r16, r32)
        note_ratio("region_encoder_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (n, a, b)
    # two identical steps: bit-identical gradients
    first = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    region_encoder_train(m, images, masks, feats, sample_points=pts).backward(torch.from_numpy(gz["grad_out"]).cuda().bfloat16())
    assert all(same_bits(first[n], p.grad) for n, p in m.named_parameters())


def test_training_forward_is_the_inference_forward(golden_dir):
    from visionllm_b200.train import region_encoder_train
    _, m, images, masks, feats, pts = golden_module(golden_dir)
    with torch.no_grad():
        want = m(images, masks, feats, sample_points=pts)
    got = region_encoder_train(m, images, masks, feats, sample_points=pts)
    assert same_bits(got.detach(), want)


# ---------------------------------------------------------------------------------------------------------------------
# the composite step with regions
# ---------------------------------------------------------------------------------------------------------------------
REG_ = 960


def region_composite():
    from test_padded_training_gpu import build_composite
    from visionllm_b200.region_encoder import B200RegionEncoder
    m = build_composite("mlp2x_gelu", False)
    torch.manual_seed(12)
    enc = B200RegionEncoder(hidden_dim=64, embed_dim=192, out_dim=256, mask_pool_type="grid_sample")
    with torch.no_grad():
        for n, p in enc.named_parameters():
            p.copy_(torch.randn_like(p) * (0.1 if p.dim() > 1 else 0.2) + (1.0 if n.endswith(("1.weight", "4.weight")) else 0.0))
    m.region_encoder = enc.to("cuda", torch.bfloat16)
    m.use_region_encoder = True
    m.reg_token_id = REG_
    m.freeze_vis_encoder()
    return m


def region_batch():
    from test_padded_training_gpu import composite_batch
    ids, mask, labels, images = composite_batch(64)
    ids[0, 100], ids[0, 120], ids[1, 110] = REG_, REG_, REG_             # 2 / 1 regions per sample
    labels[ids == REG_] = -100
    regions = [torch.zeros(2, 112, 112), torch.zeros(1, 112, 112)]      # sample 1's region: an empty mask
    regions[0][0, 10:60, 20:100] = 1
    regions[0][1, 90:93, 5:8] = 1                                        # 9 pixels
    g = torch.Generator().manual_seed(4)
    pts = []
    for lv in range(3):
        per = []
        for i, r in enumerate((regions[0][0], regions[0][1], regions[1][0])):
            nz = r.nonzero().float()
            if len(nz) and not (i == 1 and lv == 0):
                keep = torch.randperm(len(nz), generator=g)[:min(len(nz), 500)].sort()[0]
                per.append(torch.cat([torch.zeros(len(keep), 1), nz[keep] / 112], 1).cuda())
            else:                                           # the empty region; the 9-pixel region has no points on level 0
                per.append(torch.zeros(0, 3, device="cuda"))
        pts.append(per)
    return ids, mask, labels, images, [r.cuda().bfloat16() for r in regions], pts


def reference_region_features(m, images, regions, pts, dtype, params):
    """The region encoder restated in torch (F.conv2d, the LayerNorm2d formula, F.gelu, F.grid_sample) on the same points."""
    from visionllm_b200.modeling import region_encoder_inputs
    with torch.no_grad():
        _, _, outs = m.vision_hidden_state(images.cuda().bfloat16())
    ri, rm, rf = region_encoder_inputs(images.cuda().bfloat16(), regions, outs.hidden_states, None)
    enc = m.region_encoder

    def P(name, t):
        params["region_encoder." + name] = t.detach().to(dtype).requires_grad_(True)
        return params["region_encoder." + name]
    me = enc.mask_embedding
    x = torch.cat([ri, rm], 1).to(dtype)

    def ln2d(x, i):
        u = x.mean(1, keepdim=True)
        s = (x - u).pow(2).mean(1, keepdim=True)
        x = (x - u) / torch.sqrt(s + me[i].eps)
        return P(f"mask_embedding.{i}.weight", me[i].weight)[:, None, None] * x + P(f"mask_embedding.{i}.bias", me[i].bias)[:, None, None]
    x = F.conv2d(x, P("mask_embedding.0.weight", me[0].weight), P("mask_embedding.0.bias", me[0].bias), stride=7)
    x = F.gelu(ln2d(x, 1))
    x = F.conv2d(x, P("mask_embedding.3.weight", me[3].weight), P("mask_embedding.3.bias", me[3].bias), stride=2)
    x = F.gelu(ln2d(x, 4))
    x = F.conv2d(x, P("mask_embedding.6.weight", me[6].weight), P("mask_embedding.6.bias", me[6].bias))
    R, E, h, w = x.shape
    Wu, bu = P("up_dim.weight", enc.up_dim.weight), P("up_dim.bias", enc.up_dim.bias)
    outs_l = []
    for lv, f in enumerate(rf):
        x = x + f.reshape(R, h, w, -1).permute(0, 3, 1, 2).to(dtype)
        feats = []
        for r in range(R):
            p = pts[lv][r]
            if len(p) == 0:
                feats.append(torch.zeros(E, dtype=dtype, device="cuda"))
                continue
            grid = (p[:, -2:].flip(-1).to(dtype) * 2 - 1).view(1, -1, 1, 2)
            feats.append(F.grid_sample(x[r:r + 1], grid, align_corners=False).view(E, -1).mean(1))
        outs_l.append(F.linear(torch.stack(feats), Wu, bu))
    return torch.stack(outs_l).mean(0)


def reference_step_with_regions(m, ids, mask, labels, images, regions, pts, dtype):
    """test_padded_training_gpu.reference_step with the region features written at the <region> rows
    (VisionLLMv2Model.forward's order: assembly, then the region scatter, mv2.py:690-698)."""
    import test_padded_training_gpu as T
    params = {}
    feats = reference_region_features(m, images, regions, pts, dtype, params)
    orig = torch.Tensor.index_put

    def hook(emb, idx, vals, *a, **k):                                # after the image features: overwrite <region> rows
        out = orig(emb, idx, vals, *a, **k)
        if vals.shape[-1] == emb.shape[-1] and getattr(hook, "pending", False) and vals.shape[0] == (ids == T.IMP_).sum():
            hook.pending = False
            sel = torch.nonzero(ids.cuda() == REG_, as_tuple=True)
            out = orig(out, sel, feats.to(out.dtype))
        return out
    hook.pending = True
    torch.Tensor.index_put = hook
    try:
        loss, grads = T.reference_step(m, ids, mask, labels, images, dtype)
    finally:
        torch.Tensor.index_put = orig
    assert not hook.pending
    grads.update({k: v.grad for k, v in params.items()})
    return loss, grads


def test_composite_step_with_regions_matches_torch_composition():
    from visionllm_b200.train import B200VisionLLMv2ModelTrain
    m = region_composite()
    ids, mask, labels, images, regions, pts = region_batch()
    l64, g64 = reference_step_with_regions(m, ids, mask, labels, images, regions, pts, torch.float64)
    l16, g16 = reference_step_with_regions(m, ids, mask, labels, images, regions, pts, torch.bfloat16)
    tr = B200VisionLLMv2ModelTrain(m)
    kw = dict(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=images.cuda().bfloat16(), regions=regions,
              region_sample_points=pts)
    out = tr(**kw, labels=labels.clone().cuda())
    out.loss.backward()
    assert abs(float(out.loss) - l64) <= 1.5 * abs(l16 - l64) + 1e-3 * abs(l64), (float(out.loss), l64, l16)
    named = dict(m.named_parameters())
    assert any(k.startswith("region_encoder.") for k in g64)
    for n, ref in g64.items():
        got = named[n].grad
        assert got is not None, n
        a, b = rel(got, ref), rel(g16[n], ref)
        note_ratio("composite_regions_module_rule", a / (2 * b + 3e-3))
        assert a <= 2 * b + 3e-3, (n, a, b)
    assert all(p.grad is None for p in m.vis_encoder.parameters())
    assert (named["llm.model.embed_tokens.weight"].grad[REG_] == 0).all()       # <region> positions: no table gradient
    first = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}

    # two identical steps: bit-identical gradients
    m.zero_grad(set_to_none=True)
    tr(**kw, labels=labels.clone().cuda()).loss.backward()
    assert all(same_bits(first[n], p.grad) for n, p in m.named_parameters() if p.grad is not None)

    # frozen region encoder: no region gradient, every other gradient bit-identical
    m.zero_grad(set_to_none=True)
    m.freeze_region_encoder()
    tr(**kw, labels=labels.clone().cuda()).loss.backward()
    for n, p in m.named_parameters():
        if n.startswith("region_encoder."):
            assert p.grad is None, n
        elif p.grad is not None:
            assert same_bits(first[n], p.grad), n
    m.region_encoder.requires_grad_(True)

    # the production draw: no points given
    m.zero_grad(set_to_none=True)
    o = tr(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=images.cuda().bfloat16(), regions=regions,
           labels=labels.clone().cuda())
    o.loss.backward()
    assert math.isfinite(float(o.loss))
    assert all(torch.isfinite(p.grad.float()).all() for p in m.parameters() if p.grad is not None)


def test_region_training_refusals():
    from visionllm_b200.train import B200VisionLLMv2ModelTrain, region_encoder_train
    from visionllm_b200.region_encoder import B200RegionEncoder
    m = region_composite()
    m.region_encoder.mask_pool_type = "mean"
    ids, mask, labels, images, regions, pts = region_batch()
    with pytest.raises(NotImplementedError, match="grid_sample"):
        B200VisionLLMv2ModelTrain(m)(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=images.cuda().bfloat16(),
                                     regions=regions, labels=labels.cuda())
    enc = B200RegionEncoder(64, 192, 256, mask_pool_type="cross_attn").to("cuda", torch.bfloat16)
    with pytest.raises(NotImplementedError):
        region_encoder_train(enc, images.cuda().bfloat16(), regions[1][:, None], [])
