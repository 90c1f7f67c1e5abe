"""GPU parity of the wgmma GEMM + fused epilogues and the row kernels, against a plain
PyTorch fp32 reference of the same op on the same bf16-rounded inputs.

Tolerance (written here as the north-star asks): inputs are bf16 and accumulation is fp32
in both; the output is rounded to bf16 once, so |out - ref| <= 2^-8 * |ref| (one bf16 ulp)
+ 1e-3 * max|ref| (north-star's 1e-3 rel for bf16 activations, covers fp32 summation order).
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from visionllm_b200 import _lib  # noqa: E402

# tile widths under test, named by their width in 128-column units (bring-up: VLLM_TEST_GEMM_VARIANTS=1 isolates the
# 128-column tile)
TILES = {"1": _lib.GEMM_DEFAULT, "2": _lib.GEMM_WIDE_TILE}
VARIANTS = [pytest.param(TILES[t], id=t) for t in os.environ.get("VLLM_TEST_GEMM_VARIANTS", "1,2").split(",")]


def ops():
    from visionllm_b200 import ops as o
    return o


def close(out, ref, extra=1e-3):
    out = out.float(); ref = ref.float()
    tol = ref.abs() * 2.0 ** -8 + extra * ref.abs().max()
    bad = (out - ref).abs() > tol
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} off; max err {(out - ref).abs().max().item()}"


def mk(M, N, K, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(M, K, device="cuda", generator=g)).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    return x, w


SHAPES = [(128, 256, 64), (128, 256, 128), (256, 512, 256), (1025, 3200, 3200), (300, 9600, 3200), (77, 384, 256),
          (2000, 2048, 256), (1536, 4096, 4096), (513, 1376, 4096), (640, 4096, 1376), (100, 256, 2048),
          (130, 264, 72), (4100, 3200, 640), (300, 96, 48), (200, 96, 32), (4096, 288, 96), (777, 96, 384)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_plain(M, N, K, variant):
    x, w = mk(M, N, K)
    with _lib.knob("gemm_set_variant", variant):
        out = ops().linear(x, w)
        torch.cuda.synchronize()
    ref = x.float() @ w.float().T
    close(out, ref)


# the fused epilogues (bias / activation / colscale / residual / row mask, fp32 and bf16 output) are checked against
# fp64 in tests/test_gemm_epilogue_gpu.py
@pytest.mark.parametrize("variant", VARIANTS)
def test_gemm_swiglu_interleaved(variant):
    M, I, K = 300, 1376, 512
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    wg = (torch.randn(I, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    wu = (torch.randn(I, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    w = torch.stack([wg, wu], 1).reshape(2 * I, K).contiguous()
    with _lib.knob("gemm_set_variant", variant):
        out = ops().linear(x, w, act="swiglu")
    ref = torch.nn.functional.silu(x.float() @ wg.float().T) * (x.float() @ wu.float().T)
    assert out.shape == (M, I)
    close(out, ref)


def test_gemm_strided_views_and_3d():
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(4, 65, 3 * 256, device="cuda", generator=g).bfloat16()
    w = (torch.randn(512, 256, device="cuda", generator=g) / 16).bfloat16()
    xs = qkv.view(-1, 768)[:, 256:512]          # strided A (lda = 768)
    out = o.linear(xs, w)
    close(out, xs.float() @ w.float().T)
    out3 = o.linear(qkv[..., :256].contiguous(), w)
    assert out3.shape == (4, 65, 512)


def test_gemm_argument_errors():
    o = ops()
    x, w = mk(64, 64, 64)
    with pytest.raises(RuntimeError):
        o.linear(x.float(), w)
    with pytest.raises(RuntimeError):
        o.linear(x, w[:, :32])
    with pytest.raises(RuntimeError):
        o.linear(x[:, :36], w[:, :36].contiguous())      # K pitch not a multiple of 8 elements
    # SwiGLU writes bf16 only and has no column scale
    with pytest.raises(_lib.VllmB200Error, match="unsupported"):
        o.linear(x, w, act="swiglu", out_dtype=torch.float32)
    with pytest.raises(_lib.VllmB200Error, match="unsupported"):
        o.linear(x, w, act="swiglu", colscale=torch.ones(64, dtype=torch.bfloat16, device="cuda"))
    # output rows must start on 16-byte boundaries: ldc * element size % 16 != 0
    for dt, ld in ((torch.bfloat16, 68), (torch.float32, 66)):
        out = torch.empty(64, ld, dtype=dt, device="cuda")[:, :64]
        with pytest.raises(_lib.VllmB200Error, match="misaligned"):
            o.linear(x, w, out=out)
    # the C ABI: a residual pitch below n_out is invalid; row_keep is refused with SwiGLU (by ops.linear too)
    L = _lib.lib()
    c = torch.empty(64, 64, dtype=torch.bfloat16, device="cuda")
    res = torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda")
    keep = torch.ones(64, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    args = (x.data_ptr(), 64, w.data_ptr(), 64, c.data_ptr(), 64, 64, 64, 64, None, None)
    assert L.vllm_gemm_bf16(*args, res.data_ptr(), 56, 0, 0, st) == -1
    assert L.vllm_gemm_bf16_rowmask(*args, None, 0, 4, 0, keep.data_ptr(), st) == -1
    with pytest.raises(RuntimeError, match="not with swiglu"):
        o.linear(x, w, act="swiglu", row_keep=keep.bool())


@pytest.mark.parametrize("rows,cols", [(7, 3200), (1025, 3200), (300, 4096), (5, 256), (33, 12800)])
def test_rmsnorm(rows, cols):
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 3).bfloat16()
    w = (1 + 0.1 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    out = ops().rmsnorm(x, w, 1e-6)
    # reference semantics: internvit/modeling_intern_vit.py:38-44
    xf = x.float()
    n = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(torch.bfloat16)
    ref = w * n
    # same roundings in the same places: at most one bf16 ulp from rsqrt/summation order
    assert (out.float() - ref.float()).abs().max() <= 2.0 ** -7 * ref.float().abs().max()
    assert (out != ref).float().mean() < 0.02


def test_rmsnorm_strided_inplace_qk():
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(50, 3 * 3200, device="cuda", generator=g).bfloat16()
    w = torch.ones(3200, device="cuda").bfloat16()
    ref = qkv.clone()
    for s in (0, 1):
        xf = ref[:, s * 3200:(s + 1) * 3200].float()
        ref[:, s * 3200:(s + 1) * 3200] = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).bfloat16()
    for s in (0, 1):
        sl = qkv[:, s * 3200:(s + 1) * 3200]
        ops().rmsnorm(sl, w, 1e-6, out=sl)
    assert torch.equal(qkv[:, 6400:], ref[:, 6400:])
    assert (qkv.float() - ref.float()).abs().max() <= 2.0 ** -7 * ref.float().abs().max()


@pytest.mark.parametrize("rows,cols", [(100, 256), (21760, 256), (17, 1024)])
def test_layernorm(rows, cols):
    g = torch.Generator(device="cuda").manual_seed(cols)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 2 + 0.5).bfloat16()
    w = (1 + 0.1 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    out = ops().layernorm(x, w, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-5)
    close(out, ref)


def test_rope_matches_hf_formula():
    T, H, D = 77, 8, 128
    g = torch.Generator(device="cuda").manual_seed(2)
    q = torch.randn(T, H * D, device="cuda", generator=g).bfloat16()
    inv = 1.0 / (10000 ** (torch.arange(0, D, 2, device="cuda").float() / D))
    fr = torch.outer(torch.arange(T, device="cuda").float(), inv)
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos().bfloat16(), emb.sin().bfloat16()
    qh = q.view(T, H, D)
    rot = torch.cat((-qh[..., D // 2:], qh[..., :D // 2]), -1)
    ref = (qh * cos[:, None]) + (rot * sin[:, None])          # bf16 ops, like HF apply_rotary_pos_emb
    out = ops().rope_(q.clone(), cos, sin, H, D).view(T, H, D)
    assert torch.equal(out, ref)


# ---- backward GEMMs: MN-major operands (dgrad / wgrad without transposed copies) ----
@pytest.mark.parametrize("variant", [pytest.param(v, id=t) for t, v in TILES.items()])
@pytest.mark.parametrize("T,out_f,in_f", [(512, 256, 384), (2048, 4096, 4096), (300, 1376, 4096), (1000, 520, 200)])
def test_gemm_tn_dgrad_wgrad_match_torch(T, out_f, in_f, variant):
    """dx = dy . W and dW = dy^T . x through vllm_gemm_bf16_tn vs fp32 torch on the same bf16 inputs (one bf16 output
    rounding + 1e-3 max|ref|), both tile widths, ragged M / N / K tails."""
    from visionllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(T + out_f)
    dy = (torch.randn(T, out_f, device="cuda", generator=g) * 0.5).bfloat16()
    x = (torch.randn(T, in_f, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(out_f, in_f, device="cuda", generator=g) * 0.05).bfloat16()
    with _lib.knob("gemm_set_variant", variant):
        dx = ops.gemm_tn(dy, w, b_mn=True)
        dw = ops.gemm_tn(dy, x, a_mn=True, b_mn=True, out_dtype=torch.float32)
        y = ops.gemm_tn(x, w)                                            # both K-major == ops.linear
        xt = torch.zeros((in_f, (T + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")   # [K, M] with a 16-byte row pitch
        xt[:, :T] = x.t()
        at = ops.gemm_tn(xt[:, :T], w, a_mn=True)                       # MN-major A alone
    ref_dx = dy.float() @ w.float()
    ref_dw = dy.float().t() @ x.float()
    ref_y = x.float() @ w.float().t()
    for got, ref in ((dx, ref_dx), (y, ref_y), (at, ref_y)):
        assert got.shape == ref.shape
        assert ((got.float() - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-3 * ref.abs().max()).all()
    assert dw.dtype == torch.float32 and (dw - ref_dw).abs().max() <= 1e-3 * ref_dw.abs().max()
    assert torch.equal(y, ops.linear(x, w))
