"""Drop-in for the reference extension module ``MultiScaleDeformableAttention``.

Same surface as the pybind module built from
``visionllmv2/model/unipose/ops/src/vision.cpp:13-16`` (positional
``im2col_step``) and as ``mmcv._ext`` (keyword ``im2col_step``,
``mmcv/ops/multi_scale_deform_attn.py:54-94``):

    ms_deform_attn_forward(value, spatial_shapes, level_start_index,
                           sampling_loc, attn_weight, im2col_step) -> Tensor[N, Lq, M*D]

Install it where the reference looks it up::

    import visionllm_b200.msda as ext
    gd.MultiScaleDeformableAttention = ext          # grounding_dino/...mask_dn.py:110,147
    sys.modules["MultiScaleDeformableAttention"] = ext   # unipose/ops/functions/ms_deform_attn_func.py:19
    mmcv.ops.multi_scale_deform_attn.ext_module = ext    # mmcv/ops/multi_scale_deform_attn.py:19-20

Errors follow the reference's convention (RuntimeError for non-contiguous /
non-CUDA / wrong-dtype inputs and for ``batch % min(batch, im2col_step) != 0``,
ms_deform_attn_cuda.cu:215-245) -- and, unlike the reference, launch errors
raise too.  ``im2col_step`` is validated and otherwise ignored (one launch).
"""
import torch

from . import _lib

STRICT = 1

_shape_cache = {}


def attach_host_shapes(spatial_shapes, shapes_list):
    """Remember the python-side (H, W) list a device `spatial_shapes` tensor was built from, so that later consumers
    (tiling hint here, reference points / proposals in the GDINO stage) never read it back from the device -- a
    device->host copy is a sync and is illegal during CUDA-graph capture."""
    spatial_shapes._b200_host = torch.tensor([[int(h), int(w)] for h, w in shapes_list], dtype=torch.int64)
    return spatial_shapes


def host_shape_list(spatial_shapes):
    """[(H, W), ...] of a spatial_shapes tensor: the attached host copy if there is one, else a device read."""
    hs = getattr(spatial_shapes, "_b200_host", None)
    return [(int(h), int(w)) for h, w in (hs if hs is not None else spatial_shapes).tolist()]


def _host_shapes(spatial_shapes):
    """Cached host copy of the (tiny) spatial_shapes tensor: work-ordering hint only."""
    hs = getattr(spatial_shapes, "_b200_host", None)
    if hs is not None:
        return hs
    # The caching allocator recycles addresses: a new tensor can reuse a dead one's (ptr, version).  The hint only
    # orders work (the kernels read the geometry on the device), but its LENGTH must match, so the shape is in the key.
    key = (spatial_shapes.data_ptr(), spatial_shapes._version, spatial_shapes.device.index, tuple(spatial_shapes.shape))
    hit = _shape_cache.get(key)
    if hit is None:
        if len(_shape_cache) > 64:
            _shape_cache.clear()
        hit = spatial_shapes.detach().to("cpu", torch.int64).contiguous()
        _shape_cache[key] = hit
    return hit


def _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step=None, *,
                  value_dtypes=(torch.float32, torch.float64), loc_dtype=None, dtype_msg=None):
    """loc_dtype None: sampling_loc / attn_weight must have the dtype of value (the reference's rule); else they must be
    loc_dtype and a mismatch raises dtype_msg.  im2col_step None: the entry point has no such argument."""
    names = ("value", "spatial_shapes", "level_start_index", "sampling_loc", "attn_weight")
    for n, t in zip(names, (value, spatial_shapes, level_start_index, sampling_loc, attn_weight)):
        if not t.is_contiguous():
            raise RuntimeError(f"{n} tensor has to be contiguous")
        if not t.is_cuda:
            raise RuntimeError(f"{n} must be a CUDA tensor")
    if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
        raise RuntimeError("spatial_shapes / level_start_index must be int64")
    if loc_dtype is not None:
        if value.dtype not in value_dtypes or sampling_loc.dtype != loc_dtype or attn_weight.dtype != loc_dtype:
            raise RuntimeError(dtype_msg)
    elif value.dtype not in value_dtypes:
        raise RuntimeError(f"ms_deform_attn_forward not implemented for '{value.dtype}'")
    elif sampling_loc.dtype != value.dtype or attn_weight.dtype != value.dtype:
        raise RuntimeError("expected sampling_loc / attn_weight to have the dtype of value")
    if value.dim() != 4 or sampling_loc.dim() != 6 or attn_weight.dim() != 5:
        raise RuntimeError("expected value[N,S,M,D], sampling_loc[N,Lq,M,L,P,2], attn_weight[N,Lq,M,L,P]")
    N, S, M, D = value.shape
    L = spatial_shapes.shape[0]
    _, Lq, M2, L2, P, two = sampling_loc.shape
    if (M2, L2, two) != (M, L, 2) or tuple(attn_weight.shape) != (N, Lq, M, L, P) or sampling_loc.shape[0] != N:
        raise RuntimeError("inconsistent MSDA shapes")
    if im2col_step is not None:
        step = min(N, int(im2col_step)) if N > 0 else 1
        if step <= 0 or (N > 0 and N % step != 0):
            raise RuntimeError(f"batch({N}) must divide im2col_step({step})")
    return N, S, M, D, L, Lq, P


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                           im2col_step=64, *, flags=0, host_shapes=None):
    N, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                         im2col_step)
    out = torch.empty((N, Lq, M * D), dtype=value.dtype, device=value.device)
    if out.numel() == 0:
        return out
    L_ = _lib.lib()
    with torch.cuda.device(value.device):
        stream = torch.cuda.current_stream().cuda_stream
        if value.dtype == torch.float32:
            hs = host_shapes if host_shapes is not None else _host_shapes(spatial_shapes)
            rc = L_.vllm_msda_forward_f32(value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
                                          sampling_loc.data_ptr(), attn_weight.data_ptr(), out.data_ptr(),
                                          N, S, M, D, L, Lq, P, hs.data_ptr(), int(flags), stream)
        else:
            rc = L_.vllm_msda_forward_f64(value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
                                          sampling_loc.data_ptr(), attn_weight.data_ptr(), out.data_ptr(),
                                          N, S, M, D, L, Lq, P, stream)
    _lib.check(rc, "ms_deform_attn_forward")
    return out


def ms_deform_attn_sample_indices(spatial_shapes, sampling_loc):
    """(h_low, w_low, mask) int32 per sample, from the device function the kernels use."""
    if sampling_loc.dtype != torch.float32 or not sampling_loc.is_cuda or not sampling_loc.is_contiguous():
        raise RuntimeError("sampling_loc must be a contiguous CUDA float32 tensor")
    L, P = sampling_loc.shape[-3], sampling_loc.shape[-2]
    n = sampling_loc.numel() // 2
    out = torch.empty(tuple(sampling_loc.shape[:-1]) + (3,), dtype=torch.int32, device=sampling_loc.device)
    with torch.cuda.device(sampling_loc.device):
        rc = _lib.lib().vllm_msda_sample_indices_f32(spatial_shapes.data_ptr(), sampling_loc.data_ptr(),
                                                     out.data_ptr(), n, L, P,
                                                     torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ms_deform_attn_sample_indices")
    return out


def ms_deform_attn_forward_bf16(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out_dtype=None):
    """"Fast mode" (SURVEY 8d cfg 2b), an extension next to the reference API: value bf16 [N,S,M,32] read in place
    (the reference upcasts it with .float() first, gd.py:764), sampling_loc / attn_weight fp32, fp32 accumulation,
    out bf16 (default) or fp32.  The same products as ms_deform_attn_forward(value.float(), ...) summed in another
    order (bit-identical only for levels * points == 1), then one rounding to the output dtype."""
    N, S, M, D, L, Lq, P = _check_inputs(
        value, spatial_shapes, level_start_index, sampling_loc, attn_weight, value_dtypes=(torch.bfloat16,),
        loc_dtype=torch.float32,
        dtype_msg="ms_deform_attn_forward_bf16: value must be bf16, sampling_loc / attn_weight fp32")
    out_dtype = out_dtype or torch.bfloat16
    if out_dtype not in (torch.bfloat16, torch.float32):
        raise RuntimeError("out_dtype must be bf16 or fp32")
    out = torch.empty((N, Lq, M * D), dtype=out_dtype, device=value.device)
    if out.numel() == 0:
        return out
    hs = _host_shapes(spatial_shapes)
    with torch.cuda.device(value.device):
        rc = _lib.lib().vllm_msda_forward_bf16v(
            value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
            attn_weight.data_ptr(), out.data_ptr(), 1 if out_dtype == torch.bfloat16 else 0, N, S, M, D, L, Lq, P,
            hs.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ms_deform_attn_forward_bf16")
    return out


FUSED_MODULE_INPUT = True       # gdino.py: encoder-shape modules hand the packed projection output to the kernel


def ms_deform_attn_forward_fused(value, spatial_shapes, level_start_index, qp, reference_points, out_dtype=None,
                                 want_weights=True):
    """The inner part of `GroundingDinoMultiscaleDeformableAttention.forward` (gd.py:742-776) in ONE kernel for the encoder
    shape: value bf16 [N, S, M, 32], qp bf16 [N, Lq, >= 3*M*16] = packed offsets | logits of the (query-side) projection,
    reference_points fp32 [N, Lq, 4, 2].  Returns (out [N, Lq, M*32], attention_weights bf16 [N, Lq, M, 4, 4] or None), or
    None when the fused path does not apply (caller keeps the unfused torch ops + ms_deform_attn_forward_bf16) -- both
    paths give bit-identical results."""
    if not FUSED_MODULE_INPUT or value.dtype != torch.bfloat16 or qp.dtype != torch.bfloat16 or value.dim() != 4:
        return None
    N, S, M, D = value.shape
    L = spatial_shapes.shape[0]
    if (D != 32 or L != 4 or qp.dim() != 3 or qp.shape[1] != S or qp.shape[0] != N or qp.stride(2) != 1
            or qp.stride(0) != qp.shape[1] * qp.stride(1) or qp.shape[2] < M * 16 * 3
            or reference_points.shape != (N, S, L, 2) or not value.is_contiguous()):
        return None
    ref = reference_points.to(torch.float32).contiguous()
    out_dtype = out_dtype or torch.bfloat16
    out = torch.empty((N, S, M * D), dtype=out_dtype, device=value.device)
    attw = torch.empty((N, S, M, L, 4), dtype=torch.bfloat16, device=value.device) if want_weights else None
    hs = _host_shapes(spatial_shapes)
    with torch.cuda.device(value.device):
        rc = _lib.lib().vllm_msda_forward_fused_bf16(
            value.data_ptr(), level_start_index.data_ptr(), qp.data_ptr(), qp.stride(1), ref.data_ptr(), out.data_ptr(),
            1 if out_dtype == torch.bfloat16 else 0, attw.data_ptr() if attw is not None else None, N, S, M, D, L, S, 4,
            hs.data_ptr(), torch.cuda.current_stream().cuda_stream)
    if rc == -2:                                                  # VLLM_EUNSUPPORTED: window path not applicable
        return None
    _lib.check(rc, "ms_deform_attn_forward_fused")
    return out, attw


def supports_bf16_value(D, L, P):
    return D == 32 and L * P <= 32


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, *rest,
                            im2col_step=64):
    """Both reference flavours:
      unipose / HF (vision.cpp:13-16):  backward(v, shapes, lsi, loc, w, grad_out, im2col_step) -> [gv, gloc, gw]
      mmcv (pybind.cpp:793-798):        backward(v, shapes, lsi, loc, w, grad_out, gv, gloc, gw, im2col_step=) -> None
                                        with the three grads pre-zeroed by the caller
                                        (mmcv/ops/multi_scale_deform_attn.py:80-94)."""
    if len(rest) == 1:
        im2col_step, grads = rest[0], None
    elif len(rest) == 3:
        grads = rest
    elif len(rest) == 0:
        grads = None
    else:
        raise TypeError("ms_deform_attn_backward: unexpected arguments")
    N, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                         im2col_step)
    if not grad_output.is_contiguous() or grad_output.dtype != value.dtype or not grad_output.is_cuda:
        raise RuntimeError("grad_output tensor has to be a contiguous CUDA tensor of the dtype of value")
    if grad_output.numel() != N * Lq * M * D:
        raise RuntimeError("grad_output shape mismatch")
    if grads is None:
        gv, gl, gw = torch.zeros_like(value), torch.empty_like(sampling_loc), torch.empty_like(attn_weight)
    else:
        gv, gl, gw = grads
        for t, ref in ((gv, value), (gl, sampling_loc), (gw, attn_weight)):
            if t.shape != ref.shape or t.dtype != ref.dtype or not t.is_contiguous() or not t.is_cuda:
                raise RuntimeError("gradient buffers must match their inputs (shape, dtype, contiguous, CUDA)")
    if value.numel() and Lq:
        L_ = _lib.lib()
        fn = L_.vllm_msda_backward_f32 if value.dtype == torch.float32 else L_.vllm_msda_backward_f64
        with torch.cuda.device(value.device):
            rc = fn(value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
                    attn_weight.data_ptr(), grad_output.data_ptr(), gv.data_ptr(), gl.data_ptr(), gw.data_ptr(),
                    N, S, M, D, L, Lq, P, torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "ms_deform_attn_backward")
    elif grads is None:
        gl.zero_(); gw.zero_()
    return None if grads is not None else [gv, gl, gw]


class MultiScaleDeformableAttentionFunction(torch.autograd.Function):
    """Same autograd wrapper the reference defines around the extension (gd.py:135-180)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        ctx.im2col_step = im2col_step
        out = ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                                     attention_weights, im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                              attention_weights)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        v, shapes, lsi, loc, w = ctx.saved_tensors
        gv, gl, gw = ms_deform_attn_backward(v, shapes, lsi, loc, w, grad_output.contiguous(), ctx.im2col_step)
        return gv, None, None, gl, gw, None
