"""ctypes binding of libvllm_b200.so (the C-ABI in include/vllm_b200.h).

The library is built in-tree by ``make`` / ``__graft_entry__.build()`` and is
the ONLY compute path of this package: a missing library is an ImportError at
first use, never a silent fallback (the reference silently falls back to
grid_sample, grounding_dino/modeling_ov_grounding_dino_mask_dn.py:777-779).
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvllm_b200.so")

_lock = threading.Lock()
_lib = None
_launches = 0  # number of C-ABI compute calls issued (bench.py's gpu_launches)

c_i64p = ctypes.POINTER(ctypes.c_int64)
vp = ctypes.c_void_p
ci = ctypes.c_int
cll = ctypes.c_longlong
cf = ctypes.c_float

_SIGNATURES = {
    "vllm_version": (ctypes.c_char_p, []),
    "vllm_msda_forward_f32": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp, ci, vp]),
    "vllm_msda_forward_bf16v": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, vp]),
    "vllm_msda_pack_pairs_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    "vllm_msda_forward_pairs": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, vp]),
    "vllm_msda_forward_f64": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]),
    "vllm_msda_backward_f32": (ci, [vp] * 9 + [ci] * 7 + [vp]),
    "vllm_msda_backward_f64": (ci, [vp] * 9 + [ci] * 7 + [vp]),
    "vllm_msda_sample_indices_f32": (ci, [vp, vp, vp, cll, ci, ci, vp]),
    "vllm_msda_set_variant": (ci, [ci]),
    "vllm_msda_set_window": (ci, [ci, ci, ci]),
    "vllm_msda_set_window_fill": (ci, [ci]),
    "vllm_msda_forward_fused_bf16": (ci, [vp, vp, vp, ci, vp, vp, ci, vp, ci, ci, ci, ci, ci, ci, ci, vp, vp]),
    "vllm_seq_index": (ci, [vp, ci, ci, vp, vp, ci, cll, ci, cll, vp, vp, ci, vp, vp, vp, vp, vp, vp, vp]),
    "vllm_assemble_embeds_bf16": (ci, [vp] * 8 + [cll, ci, vp]),
    "vllm_text_query_gather_bf16": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp]),
    "vllm_gather_rows_bf16": (ci, [vp, cll, cll, vp, cll, ci, vp, vp]),
    "vllm_pixel_shuffle_rows_bf16": (ci, [vp, cll, cll, ci, ci, ci, ci, ci, vp, vp, cf, vp, ci, vp]),
    "vllm_sine_embed_f32": (ci, [vp, vp, vp, vp, cll, ci, cf, vp, ci, cll, vp, cll, ci, cll, cll, vp, vp]),
    "vllm_det_postprocess_f32": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp]),
    "vllm_mask_postprocess_f32": (ci, [vp, vp] + [ci] * 8 + [vp, vp]),
    "vllm_dcnv3_forward_f32": (ci, [vp, vp, vp, vp] + [ci] * 15 + [cf, ci, vp]),
    "vllm_dcnv3_backward_f32": (ci, [vp] * 7 + [ci] * 15 + [cf, vp]),
    "vllm_gemm_set_sm_limit": (ci, [ci, ci]),
    "vllm_gemm_bf16": (ci, [vp, ci, vp, ci, vp, ci, ci, ci, ci, vp, vp, vp, ci, ci, ci, vp]),
    "vllm_gemm_bf16_rowmask": (ci, [vp, ci, vp, ci, vp, ci, ci, ci, ci, vp, vp, vp, ci, ci, ci, vp, vp]),
    "vllm_conv_rows_bf16": (ci, [vp, cll, ci, ci, ci, ci, vp, ci, vp, ci, ci, vp, ci, vp]),
    "vllm_gemm_bf16_tn": (ci, [vp, ci, ci, vp, ci, ci, vp, ci, ci, ci, ci, ci, vp]),
    "vllm_gemm_bf16_batched": (ci, [vp, ci, ci, vp, ci, ci, vp, ci, ci, ci, ci, ci, ci, ci, vp]),
    "vllm_rmsnorm_bwd_bf16": (ci, [vp, cll, vp, vp, cll, vp, cll, vp, cll, ci, cf, vp]),
    "vllm_head_stack_bf16": (ci, [vp, vp, ci, ci, ci, ci, ci, ci, vp]),
    "vllm_rmsnorm_bwd_partials": (ci, [cll]),
    "vllm_rmsnorm_bwd_ws_bf16": (ci, [vp, cll, vp, vp, cll, vp, cll, vp, vp, ci, cll, ci, cf, vp]),
    "vllm_swiglu_fwd_bf16": (ci, [vp, cll, vp, cll, cll, ci, vp]),
    "vllm_swiglu_bwd_bf16": (ci, [vp, cll, vp, cll, vp, cll, cll, ci, vp]),
    "vllm_softmax_causal_bf16": (ci, [vp, cll, cll, ci, cf, vp]),
    "vllm_attn_ds_bf16": (ci, [vp, vp, cll, cll, ci, cf, vp]),
    "vllm_ce_loss_f32": (ci, [vp, cll, vp, vp, cll, ci, vp, vp, cll, vp]),
    "vllm_gemm_set_variant": (ci, [ci]),
    "vllm_gemm_set_group_m": (ci, [ci]),
    "vllm_rmsnorm_bf16": (ci, [vp, cll, vp, vp, cll, cll, ci, cf, vp]),
    "vllm_layernorm_bf16": (ci, [vp, cll, vp, vp, vp, cll, cll, ci, cf, vp]),
    "vllm_layernorm_gelu_bf16": (ci, [vp, cll, vp, vp, vp, cll, cll, ci, cf, vp]),
    "vllm_layernorm_gather_bf16": (ci, [vp, cll, vp, cll, cll, cll, vp, vp, vp, cll, ci, cf, vp]),
    "vllm_layernorm_residual_bf16": (ci, [vp, cll, vp, vp, vp, cll, vp, cll, cll, ci, cf, vp]),
    "vllm_dcnv3_prep_f32": (ci, [vp, cll, vp, vp, vp, cll, ci, ci, vp]),
    "vllm_dcnv3_blend_bf16": (ci, [vp, vp, vp, vp, cll, ci, ci, vp]),
    "vllm_dwconv_nhwc_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    "vllm_rope_bf16": (ci, [vp, cll, vp, vp, cll, ci, ci, vp]),
    "vllm_groupnorm_workspace_bytes": (cll, [ci, ci]),
    "vllm_groupnorm_nhwc_bf16": (ci, [vp, vp, vp, vp, ci, cll, ci, ci, cf, ci, vp, cll, vp]),
    "vllm_upsample_add_nhwc_bf16": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, ci, vp]),
    "vllm_upsample_add_nhwc_bf16_ex": (ci, [vp, cll, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]),
    "vllm_groupnorm_nhwc_bf16_grid": (ci, [vp, vp, vp, vp, ci, cll, cll, cll, cll, ci, ci, cf, ci, vp, cll, vp]),
    "vllm_attention_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cll, cll, cll, cll, cll, cll, cll, cll,
                                 vp, vp, vp, vp, ci, ci, cf, vp, cll, vp]),
    "vllm_attention_bf16_tiles": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cll, cll, cll, cll, cll, cll, cll, cll,
                                       vp, vp, vp, cf, vp, vp, vp]),
    "vllm_attention_mask_tiles": (ci, [vp, cll, ci, ci, vp, vp, vp]),
    "vllm_attention_set_variant": (ci, [ci]),
    "vllm_peer_alloc": (ci, [ctypes.POINTER(vp), ctypes.c_size_t]),
    "vllm_peer_free": (ci, [vp]),
    "vllm_peer_handle_bytes": (ci, []),
    "vllm_peer_export": (ci, [vp, vp]),
    "vllm_peer_open": (ci, [vp, ctypes.POINTER(vp)]),
    "vllm_peer_close": (ci, [vp]),
    "vllm_gemm_bf16_scatter": (ci, [vp, ci, vp, ci, vp, vp, ci, ci, ci, ci, ci, vp]),
    "vllm_tp_reduce_norm_bf16": (ci, [vp, ci, cll, vp, vp, cf, vp, ci, cll, vp, ctypes.c_uint, vp, ci, ci, ci, vp]),
    "vllm_tp_norm_ctas": (ci, [ci]),
    "vllm_tp_wait": (ci, [vp, ctypes.c_uint, vp]),
    "vllm_tp_signal": (ci, [vp, ci, ctypes.c_uint, vp]),
}


class VllmB200Error(RuntimeError):
    pass


def exported_symbols():
    return sorted(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise ImportError(
                        f"{LIB_PATH} is missing: build it with `make` or "
                        "`python -c 'import __graft_entry__ as g; g.build()'`. "
                        "visionllm_b200 has no CPU/eager fallback.")
                L = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(L, name)
                    fn.restype = res
                    fn.argtypes = args
                _lib = L
    return _lib


_ERR = {-1: "invalid argument", -2: "unsupported shape", -3: "misaligned pointer"}


def check(rc, what):
    """Raise on a non-zero C-ABI return code."""
    global _launches
    _launches += 1
    if rc == 0:
        return
    if rc < 0:
        raise VllmB200Error(f"{what}: {_ERR.get(rc, 'error')} (rc={rc})")
    raise VllmB200Error(f"{what}: CUDA error {rc} at launch")


def launch_count():
    return _launches


def add_launches(n):
    """Account for launches replayed from a captured CUDA graph (visionllm_b200.graphs)."""
    global _launches
    _launches += int(n)
