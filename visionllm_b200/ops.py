"""Torch-tensor front end of the C-ABI compute kernels (no math happens in Python).

Every function validates shapes/dtypes/contiguity, allocates the output with
torch (device memory is torch's job), and enqueues ONE kernel on the current
CUDA stream through ``_lib``.  No fallbacks: a failing launch raises.
"""
import torch

from . import _lib

ACT = {None: 0, "none": 0, "gelu": 1, "relu": 2, "silu": 3, "swiglu": 4, "quick_gelu": 5}

# Optional per-launch CUDA-event profile (bench.py's live roofline numbers): set PROFILE = [] to collect
# (kernel, algorithmic flops, algorithmic bytes, start_event, end_event) tuples; None = off (default).
PROFILE = None


class _Prof:
    __slots__ = ("name", "flops", "bytes", "e0", "tag")

    def __init__(self, name, flops=0.0, nbytes=0.0, tag=None):
        self.name, self.flops, self.bytes, self.tag = name, flops, nbytes, tag

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.name, self.flops, self.bytes, self.e0, e1, self.tag))
        return False


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _as_u8(t):
    """A mask for the kernels (uint8, contiguous): a bool tensor is reinterpreted in place (same bytes, 0 / 1), not copied."""
    if t.dtype == torch.bool:
        return t.contiguous().view(torch.uint8)
    return t.to(torch.uint8).contiguous()


def _bf16_2d(t, name):
    if t.dtype != torch.bfloat16 or not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA bfloat16 tensor")
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError(f"{name} must be 2-D with unit inner stride")
    return t


def linear(x, weight, bias=None, act=None, colscale=None, residual=None, out_dtype=torch.bfloat16, out=None,
           row_keep=None):
    """y = epi(x @ weight.T): x [..., K] bf16, weight [N, K] bf16 (nn.Linear layout).

    epi = (+bias) -> act -> (*colscale) -> (+residual); act='swiglu' expects gate/up rows
    interleaved in `weight` and returns N/2 columns.  One wgmma kernel launch.
    row_keep: optional bool/uint8 [...] (one per row): rows with False are stored as exact zeros
    (`masked_fill(~row_keep[..., None], 0)` folded into the epilogue).
    """
    lead = x.shape[:-1]
    K = x.shape[-1]
    x2 = x.reshape(-1, K) if x.dim() != 2 else x
    _bf16_2d(x2, "x"); _bf16_2d(weight, "weight")
    N = weight.shape[0]
    if weight.shape[1] != K:
        raise RuntimeError(f"linear: x has K={K} but weight is {tuple(weight.shape)}")
    a = ACT[act]
    n_out = N // 2 if a == 4 else N
    M = x2.shape[0]
    if out is None:
        out = torch.empty((M, n_out), dtype=out_dtype, device=x.device)
    else:
        if out.shape != (M, n_out) or out.stride(1) != 1:
            raise RuntimeError("linear: bad `out`")
        out_dtype = out.dtype
    if out_dtype not in (torch.bfloat16, torch.float32):
        raise RuntimeError("linear: out dtype must be bf16 or fp32")
    res2 = None
    if residual is not None:
        res2 = residual.reshape(-1, n_out) if residual.dim() != 2 else residual
        _bf16_2d(res2, "residual")
        if res2.shape != (M, n_out):
            raise RuntimeError("linear: residual shape mismatch")
    for v, nm in ((bias, "bias"), (colscale, "colscale")):
        if v is not None and (v.dtype != torch.bfloat16 or v.numel() != N or not v.is_contiguous()):
            raise RuntimeError(f"linear: {nm} must be contiguous bf16 [N]")
    rk = None
    if row_keep is not None:
        if row_keep.numel() != M or not row_keep.is_cuda or a == 4:
            raise RuntimeError("linear: row_keep must be a CUDA mask with one entry per row (not with swiglu)")
        rk = _as_u8(row_keep.reshape(-1))
    with torch.cuda.device(x.device), _Prof("gemm", 2.0 * M * N * K,
                                            2.0 * (M * K + N * K) + out.element_size() * M * n_out, f"{M}x{N}x{K}"):
        args = (x2.data_ptr(), x2.stride(0), weight.data_ptr(), weight.stride(0), out.data_ptr(), out.stride(0),
                M, N, K, bias.data_ptr() if bias is not None else None,
                colscale.data_ptr() if colscale is not None else None,
                res2.data_ptr() if res2 is not None else None, res2.stride(0) if res2 is not None else 0,
                a, 1 if out_dtype == torch.float32 else 0)
        if rk is None:
            rc = _lib.lib().vllm_gemm_bf16(*args, _stream())
        else:
            rc = _lib.lib().vllm_gemm_bf16_rowmask(*args, rk.data_ptr(), _stream())
    _lib.check(rc, "vllm_gemm_bf16")
    return out.reshape(*lead, n_out)


def gemm_tn(a, b, a_mn=False, b_mn=False, out_dtype=torch.bfloat16):
    """C[M, N] = sum_k A(m, k) B(n, k) on the wgmma GEMM with K-major or MN-major operands (the backward GEMMs):
    a is [M, K] (a_mn=False) or [K, M] (a_mn=True), b is [N, K] or [K, N]; 2-D bf16, unit inner stride.
      dgrad: gemm_tn(dy, W, b_mn=True)            -> dx [T, in]
      wgrad: gemm_tn(dy, x, a_mn=True, b_mn=True) -> dW [out, in]"""
    _bf16_2d(a, "a"); _bf16_2d(b, "b")
    M, K = (a.shape[1], a.shape[0]) if a_mn else a.shape
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else b.shape
    if K != Kb:
        raise RuntimeError(f"gemm_tn: reduction sizes differ ({K} vs {Kb})")
    if out_dtype not in (torch.bfloat16, torch.float32):
        raise RuntimeError("gemm_tn: out_dtype must be bf16 or fp32")
    out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    with torch.cuda.device(a.device), _Prof("gemm", 2.0 * M * N * K, 2.0 * (M * K + N * K) + out.element_size() * M * N,
                                            f"{M}x{N}x{K}"):
        rc = _lib.lib().vllm_gemm_bf16_tn(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
                                          out.data_ptr(), out.stride(0), M, N, K, 1 if out_dtype == torch.float32 else 0,
                                          _stream())
    _lib.check(rc, "vllm_gemm_bf16_tn")
    return out


def conv2d_s1_rows(x, weight_rows, bias, kernel, padding, act=None, prepadded=False):
    """Stride-1 KxK convolution of a channels-last map x [B, H, W, C] (bf16) with `weight_rows` [Cout, K*K*C] in
    (dy, dx, c) order -> [B, Ho, Wo, Cout] (a strided view of the kernel's padded-grid output).  One zero-pad copy of x,
    then ONE implicit-GEMM launch (vllm_conv_rows_bf16) -- no im2col buffer (9x the activation for a 3x3).
    prepadded: x already IS the zero-bordered [B, H + 2p, W + 2p, C] map (`upsample_add_nhwc(..., pad=p)`): no pad copy."""
    if x.dim() != 4 or x.dtype != torch.bfloat16 or not x.is_cuda:
        raise RuntimeError("conv2d_s1_rows: x must be a CUDA bf16 [B, H, W, C] tensor")
    k, p = int(kernel), int(padding)
    if prepadded:
        if not x.is_contiguous() or x.shape[1] <= 2 * p or x.shape[2] <= 2 * p:
            raise RuntimeError("conv2d_s1_rows: a prepadded x must be a contiguous [B, H + 2p, W + 2p, C] map")
        B, Hh, W, C = x.shape[0], x.shape[1] - 2 * p, x.shape[2] - 2 * p, x.shape[3]
    else:
        B, Hh, W, C = x.shape
    _bf16_2d(weight_rows, "weight_rows")
    if weight_rows.shape[1] != k * k * C:
        raise RuntimeError("conv2d_s1_rows: weight_rows must be [Cout, K*K*C]")
    Cout = weight_rows.shape[0]
    if bias is not None and (bias.dtype != torch.bfloat16 or bias.numel() != Cout or not bias.is_contiguous()):
        raise RuntimeError("conv2d_s1_rows: bias must be contiguous bf16 [Cout]")
    Hp, Wp = Hh + 2 * p, W + 2 * p
    Ho, Wo = Hp - k + 1, Wp - k + 1
    xp = x if prepadded else (torch.nn.functional.pad(x, (0, 0, p, p, p, p)) if p else x.contiguous())
    out = torch.empty((B, Hp, Wp, Cout), dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device), _Prof("gemm", 2.0 * B * Hp * Wp * Cout * k * k * C,
                                            2.0 * (B * Hp * Wp * (C + Cout) + Cout * k * k * C)):
        rc = _lib.lib().vllm_conv_rows_bf16(xp.data_ptr(), B * Hp * Wp, C, Wp, k, k, weight_rows.data_ptr(),
                                            weight_rows.stride(0), out.data_ptr(), Cout, Cout,
                                            bias.data_ptr() if bias is not None else None, ACT[act], _stream())
    _lib.check(rc, "vllm_conv_rows_bf16")
    return out[:, :Ho, :Wo]


def _rows(x, name):
    if x.dtype != torch.bfloat16 or not x.is_cuda or x.stride(-1) != 1:
        raise RuntimeError(f"{name} must be CUDA bf16 with unit inner stride")
    if x.dim() == 2:
        return x, x.shape[0], x.stride(0)
    xc = x if x.is_contiguous() else None
    if xc is None:
        raise RuntimeError(f"{name}: >2-D inputs must be contiguous")
    return xc, xc.numel() // xc.shape[-1], xc.shape[-1]


def rmsnorm(x, weight, eps, out=None):
    """apex FusedRMSNorm / InternRMSNorm / LlamaRMSNorm forward; x may be a strided 2-D view."""
    xv, rows, ldx = _rows(x, "x")
    cols = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    ov, _, ldy = _rows(out, "out")
    with torch.cuda.device(x.device), _Prof("rmsnorm", 0.0, 4.0 * rows * cols):
        rc = _lib.lib().vllm_rmsnorm_bf16(xv.data_ptr(), ldx, weight.data_ptr(), ov.data_ptr(), ldy, rows, cols,
                                          float(eps), _stream())
    _lib.check(rc, "vllm_rmsnorm_bf16")
    return out


def layernorm(x, weight, bias, eps, out=None, gelu=False, residual=None):
    """nn.LayerNorm over the last dim (bf16 rows, fp32 statistics); gelu=True appends exact-erf GELU in the same pass;
    residual (same shape) returns residual + LN(x) in the same pass."""
    xv, rows, ldx = _rows(x, "x")
    cols = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    ov, _, ldy = _rows(out, "out")
    if residual is not None:
        if gelu:
            raise RuntimeError("layernorm: gelu and residual are separate fusions")
        if residual.shape != x.shape:
            raise RuntimeError("layernorm: residual shape mismatch")
        rv, _, ldr = _rows(residual, "residual")
        with torch.cuda.device(x.device), _Prof("layernorm", 0.0, 6.0 * rows * cols):
            rc = _lib.lib().vllm_layernorm_residual_bf16(xv.data_ptr(), ldx, weight.data_ptr(), bias.data_ptr(),
                                                         rv.data_ptr(), ldr, ov.data_ptr(), ldy, rows, cols, float(eps),
                                                         _stream())
        _lib.check(rc, "vllm_layernorm_residual_bf16")
        return out
    fn = _lib.lib().vllm_layernorm_gelu_bf16 if gelu else _lib.lib().vllm_layernorm_bf16
    with torch.cuda.device(x.device), _Prof("layernorm", 0.0, 4.0 * rows * cols):
        rc = fn(xv.data_ptr(), ldx, weight.data_ptr(), bias.data_ptr(), ov.data_ptr(), ldy, rows, cols, float(eps),
                _stream())
    _lib.check(rc, "vllm_layernorm_bf16")
    return out


def layernorm_gather(x, index, weight, bias, eps):
    """out[b, j] = LN(x[b, index[j]]) (zeros where index[j] >= x.shape[1]): nn.LayerNorm + zero pad + row gather in one
    pass -- the window partition of a Swin block.  x [B, N, C] contiguous bf16, index int64 [Nout] -> [B, Nout, C]."""
    if x.dim() != 3 or x.dtype != torch.bfloat16 or not x.is_cuda or not x.is_contiguous():
        raise RuntimeError("layernorm_gather: x must be a contiguous CUDA bf16 [B, N, C] tensor")
    if index.dtype != torch.int64 or index.dim() != 1 or not index.is_cuda or not index.is_contiguous():
        raise RuntimeError("layernorm_gather: index must be a contiguous CUDA int64 vector")
    B, N, C = x.shape
    out = torch.empty((B, index.numel(), C), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device), _Prof("layernorm", 0.0, 2.0 * C * (x.shape[0] * N + out.shape[0] * out.shape[1])):
        rc = _lib.lib().vllm_layernorm_gather_bf16(x.data_ptr(), C, index.data_ptr(), N, index.numel(), B, weight.data_ptr(),
                                                   bias.data_ptr(), out.data_ptr(), C, C, float(eps), _stream())
    _lib.check(rc, "vllm_layernorm_gather_bf16")
    return out


def dcnv3_prep(packed, group, taps, with_scale):
    """packed [..., >= G*K*3 (+G)] fp32 rows (one GEMM output) -> (offset [..., G*K*2], mask [..., G*K] = softmax over
    the K taps of each group, scale [..., G] = sigmoid(logit) or None), contiguous fp32.  One launch."""
    if packed.dtype != torch.float32 or not packed.is_cuda or packed.stride(-1) != 1:
        raise RuntimeError("dcnv3_prep: packed must be CUDA fp32 with unit inner stride")
    lead = packed.shape[:-1]
    p2 = packed.reshape(-1, packed.shape[-1])
    rows = p2.shape[0]
    offset = torch.empty((*lead, group * taps * 2), dtype=torch.float32, device=packed.device)
    mask = torch.empty((*lead, group * taps), dtype=torch.float32, device=packed.device)
    scale = torch.empty((*lead, group), dtype=torch.float32, device=packed.device) if with_scale else None
    with torch.cuda.device(packed.device), _Prof("dcn_glue", 0.0, 4.0 * rows * group * taps * 6):
        rc = _lib.lib().vllm_dcnv3_prep_f32(p2.data_ptr(), p2.stride(0), offset.data_ptr(), mask.data_ptr(),
                                            scale.data_ptr() if with_scale else None, rows, group, taps, _stream())
    _lib.check(rc, "vllm_dcnv3_prep_f32")
    return offset, mask, scale


def dcnv3_blend(core, xproj, scale, group_channels):
    """bf16(core * (1 - s) + xproj * s) with s [..., G] broadcast over each group's channels (scale None: plain cast)."""
    for t in (core,) + ((xproj, scale) if scale is not None else ()):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise RuntimeError("dcnv3_blend: fp32 contiguous CUDA tensors expected")
    C = core.shape[-1]
    rows = core.numel() // C
    out = torch.empty(core.shape, dtype=torch.bfloat16, device=core.device)
    with torch.cuda.device(core.device), _Prof("dcn_glue", 0.0, 10.0 * rows * C):
        rc = _lib.lib().vllm_dcnv3_blend_bf16(core.data_ptr(), xproj.data_ptr() if scale is not None else None,
                                              scale.data_ptr() if scale is not None else None, out.data_ptr(), rows, C,
                                              int(group_channels), _stream())
    _lib.check(rc, "vllm_dcnv3_blend_bf16")
    return out


def dwconv_nhwc(x, weight_taps, bias, kernel):
    """Depthwise KxK conv (stride 1, padding K//2) of a channels-last map x [B, H, W, C] bf16; weight_taps [K*K, C]
    (the Conv2d weight [C, 1, K, K] repacked tap-major), bias [C] or None.  One launch, fp32 accumulation."""
    if x.dim() != 4 or x.dtype != torch.bfloat16 or not x.is_cuda or not x.is_contiguous():
        raise RuntimeError("dwconv_nhwc: x must be a contiguous CUDA bf16 [B, H, W, C] tensor")
    B, Hh, W, C = x.shape
    k = int(kernel)
    if weight_taps.shape != (k * k, C) or weight_taps.dtype != torch.bfloat16 or not weight_taps.is_contiguous():
        raise RuntimeError("dwconv_nhwc: weight_taps must be contiguous bf16 [K*K, C]")
    if bias is not None and (bias.dtype != torch.bfloat16 or bias.numel() != C or not bias.is_contiguous()):
        raise RuntimeError("dwconv_nhwc: bias must be contiguous bf16 [C]")
    y = torch.empty_like(x)
    with torch.cuda.device(x.device), _Prof("dwconv", 2.0 * x.numel() * k * k, 4.0 * x.numel()):
        rc = _lib.lib().vllm_dwconv_nhwc_bf16(x.data_ptr(), weight_taps.data_ptr(),
                                              bias.data_ptr() if bias is not None else None, y.data_ptr(), B, Hh, W, C,
                                              k, _stream())
    _lib.check(rc, "vllm_dwconv_nhwc_bf16")
    return y


_GN_WS = {}            # (device, stream) -> scratch: two streams running GroupNorm concurrently never share a buffer


def _ws_key(device):
    return (device.index, torch.cuda.current_stream(device).cuda_stream)


def groupnorm_nhwc(x, weight, bias, groups, eps, relu=False):
    """GroupNorm of channels-last rows x [batch, pixels, channels] (bf16), optional fused ReLU -- nn.GroupNorm(32, 256)
    of the Grounding-DINO neck (modeling_ov_grounding_dino_mask_dn.py:2085-2110) without leaving the GEMM's layout.
    x may also be a 4-D [batch, H, W, channels] VIEW of a padded grid (unit channel stride, pixel stride == channels, any row /
    image pitch: `conv2d_s1_rows`' output): the corner is read in place.  Returns contiguous [batch, pixels, channels]."""
    if x.dtype != torch.bfloat16 or not x.is_cuda or x.dim() not in (3, 4):
        raise RuntimeError("groupnorm_nhwc: x must be a CUDA bf16 [batch, pixels, channels] or [batch, H, W, channels] tensor")
    c = x.shape[-1]
    if x.dim() == 3:
        if not x.is_contiguous():
            raise RuntimeError("groupnorm_nhwc: 3-D x must be contiguous")
        n, h, w = x.shape[0], 1 if x.shape[1] else 0, x.shape[1]
        w_pitch = img_pitch = x.shape[1]
    else:
        n, h, w = x.shape[:3]
        if x.stride(3) != 1 or x.stride(2) != c or x.stride(1) % c or x.stride(0) % c:
            raise RuntimeError("groupnorm_nhwc: 4-D x must be a channels-last view with whole-pixel row / image pitches")
        w_pitch, img_pitch = x.stride(1) // c, x.stride(0) // c
    if weight.dtype != torch.bfloat16 or bias.dtype != torch.bfloat16 or weight.numel() != c or bias.numel() != c:
        raise RuntimeError("groupnorm_nhwc: weight/bias must be bf16 [channels]")
    need = _lib.lib().vllm_groupnorm_workspace_bytes(n, groups)
    key = _ws_key(x.device)
    ws = _GN_WS.get(key)
    if ws is None or ws.numel() < need:
        ws = _GN_WS[key] = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=x.device)
    out = torch.empty((n, h * w, c), dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device), _Prof("groupnorm", 0.0, 6.0 * n * h * w * c):
        rc = _lib.lib().vllm_groupnorm_nhwc_bf16_grid(x.data_ptr(), out.data_ptr(), weight.data_ptr(), bias.data_ptr(), n, h, w,
                                                      w_pitch, img_pitch, c, groups, float(eps), int(bool(relu)), ws.data_ptr(),
                                                      ws.numel(), _stream())
    _lib.check(rc, "vllm_groupnorm_nhwc_bf16_grid")
    return out


def upsample_add_nhwc(top, lateral, pad=0):
    """lateral + F.interpolate(top, size=lateral's (H, W), mode='bilinear', align_corners=False) for channels-last bf16
    maps top [B, Hi, Wi, C] (each image contiguous, any batch pitch), lateral [B, Ho, Wo, C] (the FPN top-down step,
    gd.py:2486-2492) in one pass.  pad > 0: returns the zero-bordered [B, Ho + 2 pad, Wo + 2 pad, C] map with the sum in its
    interior (the next 3x3 convolution's padded input, `conv2d_s1_rows(..., prepadded=True)`)."""
    for t, nm in ((top, "top"), (lateral, "lateral")):
        if t.dim() != 4 or t.dtype != torch.bfloat16 or not t.is_cuda:
            raise RuntimeError(f"upsample_add_nhwc: {nm} must be a CUDA bf16 [B, H, W, C] tensor")
    B, Hi, Wi, C = top.shape
    if not lateral.is_contiguous() or not top[0].is_contiguous() or (B > 1 and top.stride(0) < Hi * Wi * C):
        raise RuntimeError("upsample_add_nhwc: lateral must be contiguous, top contiguous per image")
    if lateral.shape[0] != B or lateral.shape[3] != C:
        raise RuntimeError("upsample_add_nhwc: batch / channel mismatch")
    Ho, Wo = lateral.shape[1], lateral.shape[2]
    pad = int(pad)
    out = torch.zeros((B, Ho + 2 * pad, Wo + 2 * pad, C), dtype=torch.bfloat16, device=top.device) if pad else torch.empty_like(lateral)
    with torch.cuda.device(top.device), _Prof("upsample_add", 0.0, 2.0 * (top.numel() + 2 * lateral.numel())):
        rc = _lib.lib().vllm_upsample_add_nhwc_bf16_ex(top.data_ptr(), top.stride(0) if B > 1 else Hi * Wi * C, lateral.data_ptr(),
                                                       out.data_ptr(), B, Hi, Wi, Ho, Wo, C, pad, _stream())
    _lib.check(rc, "vllm_upsample_add_nhwc_bf16_ex")
    return out


def rope_(x, cos, sin, heads, head_dim):
    """In-place rotate-half RoPE on x [tokens, >= heads*head_dim] (2-D, possibly a strided slice)."""
    if x.dim() != 2 or x.dtype != torch.bfloat16 or x.stride(1) != 1:
        raise RuntimeError("rope_: x must be 2-D bf16 with unit inner stride")
    tokens = x.shape[0]
    if tuple(cos.shape) != (tokens, head_dim) or tuple(sin.shape) != (tokens, head_dim):
        raise RuntimeError("rope_: cos/sin must be [tokens, head_dim]")
    if cos.dtype != torch.bfloat16 or not cos.is_contiguous() or not sin.is_contiguous():
        raise RuntimeError("rope_: cos/sin must be contiguous bf16")
    with torch.cuda.device(x.device), _Prof("rope", 0.0, 4.0 * tokens * heads * head_dim):
        rc = _lib.lib().vllm_rope_bf16(x.data_ptr(), x.stride(0), cos.data_ptr(), sin.data_ptr(), tokens, heads,
                                       head_dim, _stream())
    _lib.check(rc, "vllm_rope_bf16")
    return x


_ATTN_WS = {}          # (device, stream) -> split-KV scratch (grow-only), see vllm_attention_bf16


def _attn_workspace(device, nbytes):
    key = _ws_key(device)
    ws = _ATTN_WS.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _ATTN_WS[key] = ws
    return ws


class MaskTiles:
    """Live-tile lists of a sparse attention mask (`attention_mask_tiles`): the uint8 mask itself plus, per (batch*heads,
    64-row query block), the 64-key tiles with at least one allowed pair."""
    __slots__ = ("mask", "counts", "lists")

    def __init__(self, mask, counts, lists):
        self.mask, self.counts, self.lists = mask, counts, lists


def attention_mask_tiles(attn_mask):
    """attn_mask [B*H, Tq, Tk] bool / uint8, True = attend -> MaskTiles for `attention(..., attn_mask=<MaskTiles>)`: the dense
    kernel then walks only the key tiles that are not fully blocked (bit-identical result; UniPose's 50 x 69-query group mask
    is > 95 % blocked)."""
    if attn_mask.dim() != 3 or not attn_mask.is_cuda:
        raise RuntimeError("attention_mask_tiles: attn_mask must be a CUDA [B*H, Tq, Tk] tensor")
    m = _as_u8(attn_mask)
    BH, Tq, Tk = m.shape
    nqb, nkt = (Tq + 63) // 64, (Tk + 63) // 64
    counts = torch.empty((BH, nqb), dtype=torch.int32, device=m.device)
    lists = torch.empty((BH, nqb, nkt), dtype=torch.int32, device=m.device)
    with torch.cuda.device(m.device):
        rc = _lib.lib().vllm_attention_mask_tiles(m.data_ptr(), BH, Tq, Tk, counts.data_ptr(), lists.data_ptr(), _stream())
    _lib.check(rc, "vllm_attention_mask_tiles")
    return MaskTiles(m, counts, lists)


def attention(q, k, v, causal=False, scale=None, seqlens=None, key_mask=None, attn_mask=None, attn_bias=None, out=None):
    """softmax(q k^T * scale) v.  q [B, Tq, H, D], k/v [B, Tk, Hkv, D] bf16 views whose last two dims are
    contiguous (any batch/token pitch, e.g. slices of a packed qkv tensor).  Returns [B, Tq, H*D].
    seqlens: int32 [B] key lengths; key_mask: bool/uint8 [B, Tk], True = attend (arbitrary key padding);
    attn_mask: bool/uint8 [B*H, Tq, Tk], True = attend (nn.MultiheadAttention's attn_mask, inverted);
    attn_bias: fp32 [nB, H, Tq, Tk] added to the scaled scores, batch b uses slab b % nB (Swin windows)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if t.dtype != torch.bfloat16 or not t.is_cuda or t.dim() != 4:
            raise RuntimeError(f"attention: {nm} must be a 4-D CUDA bf16 tensor")
        if t.stride(3) != 1 or t.stride(2) != t.shape[3]:
            raise RuntimeError(f"attention: {nm} must have contiguous (heads, head_dim)")
    B, Tq, H, D = q.shape
    Tk, Hkv = k.shape[1], k.shape[2]
    if k.shape != v.shape or k.shape[0] != B or k.shape[3] != D or H % Hkv:
        raise RuntimeError("attention: inconsistent q/k/v shapes")
    if out is None:
        out = torch.empty((B, Tq, H * D), dtype=torch.bfloat16, device=q.device)
    if scale is None:
        scale = D ** -0.5
    sl = None
    if seqlens is not None:
        if seqlens.dtype != torch.int32 or seqlens.numel() != B or not seqlens.is_cuda:
            raise RuntimeError("attention: seqlens must be CUDA int32 [B]")
        sl = seqlens.data_ptr()
    km = None
    if key_mask is not None:
        if key_mask.shape != (B, Tk) or not key_mask.is_cuda:
            raise RuntimeError("attention: key_mask must be CUDA [B, Tk]")
        key_mask = _as_u8(key_mask)
        km = key_mask.data_ptr()
    amp, tiles = None, None
    if isinstance(attn_mask, MaskTiles):
        tiles, attn_mask = attn_mask, attn_mask.mask
        if causal or attn_bias is not None or D not in (32, 64, 128):
            raise RuntimeError("attention: a MaskTiles mask needs a non-causal call without attn_bias, head_dim 32 / 64 / 128")
    if attn_mask is not None:
        if attn_mask.shape != (B * H, Tq, Tk) or not attn_mask.is_cuda:
            raise RuntimeError("attention: attn_mask must be CUDA [B*H, Tq, Tk]")
        attn_mask = _as_u8(attn_mask)
        amp = attn_mask.data_ptr()
    abp, nb = None, 0
    if attn_bias is not None:
        if (attn_bias.dim() != 4 or tuple(attn_bias.shape[1:]) != (H, Tq, Tk) or attn_bias.dtype != torch.float32
                or not attn_bias.is_cuda or not attn_bias.is_contiguous()):
            raise RuntimeError("attention: attn_bias must be a contiguous CUDA fp32 [nB, H, Tq, Tk] tensor")
        abp, nb = attn_bias.data_ptr(), attn_bias.shape[0]
    ws_ptr, ws_bytes = None, 0
    if not causal and Tq <= 1024 and Tk >= 16 * 32:          # few queries, many keys: let the kernel split the keys
        ws_bytes = min(B * H * 64 * Tq * (D + 2) * 4, 256 << 20)
        ws_ptr = _attn_workspace(q.device, ws_bytes).data_ptr()
    fl = 4.0 * B * H * Tq * Tk * D * (0.5 if causal and Tq == Tk else 1.0)
    if tiles is not None:
        with torch.cuda.device(q.device), _Prof("attention", fl, 2.0 * B * D * (2 * Tq * H + 2 * Tk * Hkv)):
            rc = _lib.lib().vllm_attention_bf16_tiles(
                q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, Tq, Tk, H, Hkv, D,
                q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
                out.stride(0), out.stride(1), sl, km, amp, float(scale), tiles.counts.data_ptr(), tiles.lists.data_ptr(), _stream())
        _lib.check(rc, "vllm_attention_bf16_tiles")
        return out
    with torch.cuda.device(q.device), _Prof("attention", fl, 2.0 * B * D * (2 * Tq * H + 2 * Tk * Hkv)):
        rc = _lib.lib().vllm_attention_bf16(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, Tq, Tk, H, Hkv, D,
            q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
            out.stride(0), out.stride(1), sl, km, amp, abp, nb, 1 if causal else 0, float(scale), ws_ptr, ws_bytes, _stream())
    _lib.check(rc, "vllm_attention_bf16")
    return out


# ---- sequence assembly (csrc/seqglue.cu): integer index work of VisionLLMv2Model.forward as kernels -----------------
class SeqPlan:
    """Device-side result of `seq_index`: rewritten ids, per-position embedding source, [EMB] position lists."""
    __slots__ = ("new_ids", "kind", "row", "emb_pos", "emb_count", "status", "B", "L")


def seq_index(input_ids, det_tools, pose_tools, emb_token_id, num_embs, imp_token_id, split_sizes=None, tokens_per_tile=0):
    """modeling_visionllmv2.py:426-486 ([EMB] overwrite), :582-605 (<im_patch> -> ViT token map), :776-787 ([EMB] position
    lists) from ONE kernel over input_ids [B, L] (CUDA int64).  split_sizes: tiles per sample (None = one per sample) when
    image features will be scattered, or `False` for text-only."""
    if input_ids.dtype != torch.int64 or not input_ids.is_cuda or input_ids.dim() != 2:
        raise RuntimeError("seq_index: input_ids must be a CUDA int64 [B, L] tensor")
    ids = input_ids.contiguous()
    B, L = ids.shape
    dev = ids.device
    tools = [(int(t), 0) for t in det_tools if t is not None and t >= 0] + \
            [(int(t), 1) for t in pose_tools if t is not None and t >= 0]
    import ctypes
    tid = (ctypes.c_int64 * max(1, len(tools)))(*[t for t, _ in tools])
    ttb = (ctypes.c_int * max(1, len(tools)))(*[k for _, k in tools])
    p = SeqPlan()
    p.B, p.L = B, L
    p.new_ids = torch.empty_like(ids)
    p.kind = torch.empty((B, L), dtype=torch.uint8, device=dev)
    p.row = torch.empty((B, L), dtype=torch.int32, device=dev)
    p.emb_pos = torch.empty((B, L), dtype=torch.int32, device=dev)
    p.emb_count = torch.empty((B,), dtype=torch.int32, device=dev)
    p.status = torch.zeros((1,), dtype=torch.int32, device=dev)
    ts = tc = None
    if split_sizes is not False:
        sizes = [1] * B if split_sizes is None else [int(s) for s in split_sizes]
        starts = [0]
        for s in sizes[:-1]:
            starts.append(starts[-1] + s)
        meta = torch.tensor([starts, sizes], dtype=torch.int32).to(dev, non_blocking=True)
        ts, tc = meta[0], meta[1]
    with torch.cuda.device(dev):
        rc = _lib.lib().vllm_seq_index(
            ids.data_ptr(), B, L, ctypes.cast(tid, ctypes.c_void_p), ctypes.cast(ttb, ctypes.c_void_p), len(tools),
            int(emb_token_id), int(num_embs), int(imp_token_id if imp_token_id is not None else -1),
            ts.data_ptr() if ts is not None else None, tc.data_ptr() if tc is not None else None, int(tokens_per_tile),
            p.new_ids.data_ptr(), p.kind.data_ptr(), p.row.data_ptr(), p.emb_pos.data_ptr(), p.emb_count.data_ptr(),
            p.status.data_ptr(), _stream())
    _lib.check(rc, "vllm_seq_index")
    return p


def assemble_embeds(plan, embed_tokens, emb_det, emb_pose, image_features=None, base_embeds=None):
    """inputs_embeds [B, L, C] bf16 in one pass from the plan's sources (token table / caller's inputs_embeds, the two
    [EMB] tables, the ViT image tokens [rows, C])."""
    C = embed_tokens.shape[1] if embed_tokens is not None else base_embeds.shape[-1]
    srcs = [embed_tokens, emb_det, emb_pose, image_features, base_embeds]
    for t in srcs:
        if t is not None and (t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous() or t.shape[-1] != C):
            raise RuntimeError("assemble_embeds: sources must be contiguous CUDA bf16 tensors with the same hidden size")
    out = torch.empty((plan.B, plan.L, C), dtype=torch.bfloat16, device=plan.kind.device)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    with torch.cuda.device(out.device), _Prof("seq_assemble", 0.0, 4.0 * plan.B * plan.L * C):
        rc = _lib.lib().vllm_assemble_embeds_bf16(plan.kind.data_ptr(), plan.row.data_ptr(), *[ptr(t) for t in srcs],
                                                  out.data_ptr(), plan.B * plan.L, C, _stream())
    _lib.check(rc, "vllm_assemble_embeds_bf16")
    return out


def text_query_gather(plan, hidden, num_embs, max_patches):
    """mv2.py:776-787: ([B, mx, num_embs, C] bf16 zero padded, [B, mx] bool) from the [EMB] rows of `hidden` [B, L, C]."""
    if hidden.dtype != torch.bfloat16 or not hidden.is_contiguous() or hidden.shape[:2] != (plan.B, plan.L):
        raise RuntimeError("text_query_gather: hidden must be a contiguous bf16 [B, L, C] tensor")
    C = hidden.shape[2]
    tq = torch.empty((plan.B, max_patches, num_embs, C), dtype=torch.bfloat16, device=hidden.device)
    tm = torch.empty((plan.B, max_patches), dtype=torch.bool, device=hidden.device)
    with torch.cuda.device(hidden.device):
        rc = _lib.lib().vllm_text_query_gather_bf16(hidden.data_ptr(), plan.emb_pos.data_ptr(), plan.emb_count.data_ptr(),
                                                    plan.B, plan.L, C, int(num_embs), int(max_patches), tq.data_ptr(),
                                                    tm.data_ptr(), _stream())
    _lib.check(rc, "vllm_text_query_gather_bf16")
    return tq, tm


def sine_embed(feats, stride, dim_t, rows, pre_scale=0.0, out=None, out_dtype=torch.float32, add_row=None):
    """out[r, f * nd + d] = (sin | cos by parity of d)((feats[f][r * stride] * pre_scale) / dim_t[d]) -- the sine position
    embeddings of the GDINO stage in one launch (csrc/posembed.cu).  feats: 1..4 fp32 CUDA tensors addressed as
    base + r * stride (columns of one [rows, k] tensor, or contiguous maps); dim_t fp32 [nd]; out (optional): where to write,
    fp32 or bf16 with unit inner stride -- a 2-D [rows, nfeat * nd] view, or a 3-D [B, rows / B, nfeat * nd] view (one level's
    slab of a [B, S, C] buffer); add_row: bf16 [nfeat * nd] added after the bf16 rounding (the level embedding)."""
    nf, nd = len(feats), dim_t.numel()
    if not 1 <= nf <= 4 or any(f.dtype != torch.float32 or not f.is_cuda for f in feats):
        raise RuntimeError("sine_embed: 1..4 CUDA fp32 feature tensors")
    if dim_t.dtype != torch.float32 or not dim_t.is_contiguous():
        raise RuntimeError("sine_embed: dim_t must be contiguous fp32")
    if out is None:
        out = torch.empty((rows, nf * nd), dtype=out_dtype, device=feats[0].device)
    if out.dim() not in (2, 3) or out.numel() != rows * nf * nd or out.shape[-1] != nf * nd or out.stride(-1) != 1 or \
            out.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("sine_embed: out must be [rows, nfeat * nd] or [B, rows / B, nfeat * nd], fp32 / bf16, unit inner stride")
    if add_row is not None and (add_row.dtype != torch.bfloat16 or add_row.numel() != nf * nd or not add_row.is_contiguous()):
        raise RuntimeError("sine_embed: add_row must be contiguous bf16 [nfeat * nd]")
    rpb, obs, ldo = (0, 0, out.stride(0)) if out.dim() == 2 else (out.shape[1], out.stride(0), out.stride(1))
    ptr = [f.data_ptr() for f in feats] + [None] * (4 - nf)
    with torch.cuda.device(out.device), _Prof("sine_embed", 0.0, float(out.numel() * out.element_size())):
        rc = _lib.lib().vllm_sine_embed_f32(ptr[0], ptr[1], ptr[2], ptr[3], int(stride), nf, float(pre_scale), dim_t.data_ptr(), nd,
                                            int(rows), out.data_ptr(), int(ldo), int(out.dtype == torch.bfloat16), int(rpb),
                                            int(obs), None if add_row is None else add_row.data_ptr(), _stream())
    _lib.check(rc, "vllm_sine_embed_f32")
    return out


def ce_loss(logits, labels):
    """`CrossEntropyLoss()(logits.view(-1, V), labels.view(-1))` of modeling_visionllmv2.py:750-756, forward only: fp32
    logits [rows, V] (unit inner stride, any row pitch), int64 labels [rows] (-100 = ignore) -> fp32 scalar, the mean over
    the non-ignored rows (nan when every row is ignored, like torch).  One pass of `ce_loss_kernel` (csrc/train_ops.cu)."""
    if logits.dtype != torch.float32 or not logits.is_cuda or logits.dim() != 2 or logits.stride(1) != 1:
        raise RuntimeError("ce_loss: logits must be a CUDA fp32 [rows, V] matrix with unit inner stride")
    if labels.dtype != torch.int64 or not labels.is_cuda or labels.numel() != logits.shape[0]:
        raise RuntimeError("ce_loss: labels must be CUDA int64 [rows]")
    labels = labels.reshape(-1).contiguous()
    rows, V = logits.shape
    loss_sum = torch.zeros(1, dtype=torch.float32, device=logits.device)
    with torch.cuda.device(logits.device), _Prof("ce_loss", 0.0, 4.0 * rows * V):
        rc = _lib.lib().vllm_ce_loss_f32(logits.data_ptr(), logits.stride(0), labels.data_ptr(), None, rows, V,
                                         loss_sum.data_ptr(), None, 0, _stream())
    _lib.check(rc, "vllm_ce_loss_f32")
    n_valid = ((labels >= 0) & (labels < V)).sum()
    return (loss_sum / n_valid.float()).reshape(())


def gather_rows(src, idx):
    """dst[i] = src[idx[i]]: src [rows, C] bf16 (unit inner stride), idx int64 [n] (negative = from the end)."""
    _bf16_2d(src, "src")
    if idx.dtype != torch.int64 or not idx.is_cuda or not idx.is_contiguous():
        raise RuntimeError("gather_rows: idx must be a contiguous CUDA int64 tensor")
    out = torch.empty((idx.numel(), src.shape[1]), dtype=torch.bfloat16, device=src.device)
    with torch.cuda.device(src.device):
        rc = _lib.lib().vllm_gather_rows_bf16(src.data_ptr(), src.stride(0), src.shape[0], idx.data_ptr(), idx.numel(),
                                              src.shape[1], out.data_ptr(), _stream())
    _lib.check(rc, "vllm_gather_rows_bf16")
    return out


def pixel_shuffle_rows(hidden, skip_tokens, ln_weight=None, ln_bias=None, eps=1e-5, grid=None, order=0):
    """mv2.py:381-392 + :574-579 in one pass: ViT hidden state [tiles, skip + gw*gh, C] (bf16) -> [tiles, gw*gh/4, 4C], the
    CLS slice and both permute copies folded in; with (ln_weight, ln_bias) also the LayerNorm(4C) that opens `internvl_mlp`.
    grid=(rows, cols) for non-square token grids; order=1 gives HF SwinPatchMerging's concatenation order."""
    if hidden.dtype != torch.bfloat16 or not hidden.is_cuda or hidden.dim() != 3 or hidden.stride(2) != 1:
        raise RuntimeError("pixel_shuffle_rows: hidden must be a CUDA bf16 [tiles, tokens, C] tensor with unit inner stride")
    tiles, T, C = hidden.shape
    if grid is None:
        g = int(round((T - skip_tokens) ** 0.5))
        grid = (g, g)
    gw, gh = int(grid[0]), int(grid[1])
    if gw * gh != T - skip_tokens or gw % 2 or gh % 2:
        raise RuntimeError("pixel_shuffle_rows: the patch tokens must form an even grid")
    out = torch.empty((tiles, gw * gh // 4, 4 * C), dtype=torch.bfloat16, device=hidden.device)
    for t in (ln_weight, ln_bias):
        if t is not None and (t.dtype != torch.bfloat16 or t.numel() != 4 * C or not t.is_contiguous()):
            raise RuntimeError("pixel_shuffle_rows: LayerNorm weight / bias must be contiguous bf16 [4C]")
    with torch.cuda.device(hidden.device), _Prof("pixel_shuffle", 0.0, 4.0 * out.numel()):
        rc = _lib.lib().vllm_pixel_shuffle_rows_bf16(
            hidden.data_ptr(), hidden.stride(0), hidden.stride(1), int(skip_tokens), tiles, gw, gh, C,
            ln_weight.data_ptr() if ln_weight is not None else None, ln_bias.data_ptr() if ln_bias is not None else None,
            float(eps), out.data_ptr(), int(order), _stream())
    _lib.check(rc, "vllm_pixel_shuffle_rows_bf16")
    return out
