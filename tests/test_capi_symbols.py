"""CPU: the C-ABI library loads and exports every symbol include/*.h declares
(no compute calls -- there is no GPU here)."""
import ctypes
import glob
import os
import re

from visionllm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        src = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        names.update(re.findall(r"\b(vllm_\w+)\s*\(", src))
    return sorted(names)


def test_header_declares_something():
    assert "vllm_msda_forward_f32" in declared_symbols()


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_lib.LIB_PATH), "run `make` (or __graft_entry__.build()) first"
    L = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(L, s)]
    assert not missing, missing


def test_python_binding_covers_the_header():
    assert set(declared_symbols()) == set(_lib.exported_symbols())


def test_version_string():
    assert b"sm_90a" in _lib.lib().vllm_version()


def test_round2_entry_points_marshal_and_accept_empty_problems():
    """Every round-2 entry point called through the ctypes binding with an EMPTY problem (returns before any launch) and
    with a malformed one (negative error code): checks the Python-side signatures against the library without a GPU."""
    L = _lib.lib()
    assert L.vllm_msda_set_window(0, 0, 0) == 0 and L.vllm_msda_set_window(-1, 0, 0) < 0
    assert L.vllm_det_postprocess_f32(None, None, None, 0, 100, 80, 256, 100, None, None, None, None, None, None) == 0
    assert L.vllm_det_postprocess_f32(None, None, None, 1, 100, 80, 40, 100, None, None, None, None, None, None) < 0   # ld < K
    assert L.vllm_mask_postprocess_f32(None, None, 0, 64, 64, 4, 250, 250, 480, 500, None, None) == 0
    assert L.vllm_mask_postprocess_f32(None, None, 1, 64, 64, 4, 250, 250, 480, 500, None, None) < 0               # null pointers
    assert L.vllm_seq_index(None, 0, 128, None, None, 0, 32010, 4, 32002, None, None, 0, None, None, None, None, None, None, None) == 0
    assert L.vllm_seq_index(None, 1, 128, None, None, 9, 32010, 4, 32002, None, None, 0, None, None, None, None, None, None, None) < 0
    assert L.vllm_assemble_embeds_bf16(None, None, None, None, None, None, None, None, 0, 4096, None) == 0
    assert L.vllm_sine_embed_f32(None, None, None, None, 1, 2, 0.0, None, 128, 0, None, 256, 1, 0, 0, None, None) == 0
    assert L.vllm_groupnorm_nhwc_bf16_grid(None, None, None, None, 0, 8, 8, 10, 100, 256, 32, 1e-5, 0, None, 0, None) == 0
    assert L.vllm_groupnorm_nhwc_bf16_grid(None, None, None, None, 1, 8, 8, 10, 100, 256, 32, 1e-5, 0, None, 0, None) < 0   # null pointers
    assert L.vllm_upsample_add_nhwc_bf16_ex(None, 64 * 256, None, None, 0, 8, 8, 16, 16, 256, 1, None) == 0
    assert L.vllm_attention_mask_tiles(None, 0, 100, 100, None, None, None) == 0
    assert L.vllm_attention_mask_tiles(None, 4, 100, 100, None, None, None) < 0                                              # null pointers
    args = [None] * 4 + [0, 64, 64, 8, 8, 32] + [0] * 8 + [None, None, None, 1.0]
    assert L.vllm_attention_bf16_tiles(*args, None, None, None) < 0                                                          # no tile lists
    assert L.vllm_upsample_add_nhwc_bf16_ex(None, 10, None, None, 1, 8, 8, 16, 16, 256, 1, None) < 0                       # pitch < image
    assert L.vllm_sine_embed_f32(None, None, None, None, 1, 5, 0.0, None, 128, 0, None, 1024, 1, 0, 0, None, None) < 0    # > 4 features
    assert L.vllm_sine_embed_f32(None, None, None, None, 1, 2, 0.0, None, 100, 0, None, 256, 1, 0, 0, None, None) < 0     # nd % 8
    assert L.vllm_assemble_embeds_bf16(None, None, None, None, None, None, None, None, 4, 4097, None) < 0          # hidden % 8
    assert L.vllm_text_query_gather_bf16(None, None, None, 2, 128, 4096, 4, 0, None, None, None) == 0
    assert L.vllm_gather_rows_bf16(None, 4096, 10, None, 0, 4096, None, None) == 0
    assert L.vllm_pixel_shuffle_rows_bf16(None, 0, 0, 1, 0, 32, 32, 3200, None, None, 1e-5, None, 0, None) == 0
    assert L.vllm_pixel_shuffle_rows_bf16(None, 0, 0, 1, 1, 31, 32, 3200, None, None, 1e-5, None, 0, None) < 0     # odd grid
    assert L.vllm_gemm_bf16_tn(None, 64, 0, None, 64, 1, None, 64, 0, 64, 64, 0, None) == 0
    assert L.vllm_gemm_bf16_tn(None, 8, 0, None, 64, 1, None, 64, 16, 64, 64, 0, None) < 0
    assert L.vllm_gemm_bf16_batched(None, 128, 0, None, 128, 0, None, 2048, 0, 2048, 2048, 128, 1, 0, None) == 0
    assert L.vllm_gemm_bf16_batched(None, 128, 0, None, 128, 0, None, 2048, 2, 2048, 2048, 128, 7, 0, None) < 0   # causal mode
    assert L.vllm_rmsnorm_bwd_bf16(None, 4096, None, None, 4096, None, 4096, None, 0, 4096, 1e-5, None) == 0
    assert L.vllm_swiglu_fwd_bf16(None, 22016, None, 11008, 0, 11008, None) == 0
    assert L.vllm_swiglu_bwd_bf16(None, 22016, None, 11008, None, 22016, 0, 11008, None) == 0
    assert L.vllm_softmax_causal_bf16(None, 2048, 0, 2048, 0.088, None) == 0
    assert L.vllm_attn_ds_bf16(None, None, 2048, 0, 2048, 0.088, None) == 0
    assert L.vllm_ce_loss_f32(None, 32028, None, None, 0, 32026, None, None, 32032, None) == 0
