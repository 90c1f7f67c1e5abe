"""Golden vectors for tests/test_msda_gpu.py::test_forward_matches_the_reference_cuda_kernel: the outputs of the
REFERENCE's own MSDA CUDA extension (built by oracle/build_msda_ref.py into oracle/_ref/msda) on the seeded cases the test
rebuilds for itself -- forward in fp32 and fp64, the three backward gradients in fp64.  Needs a GPU and that extension.

    python tests/golden/gen_golden_msda_ref_kernel.py [output directory, default tests/golden]
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import test_msda_gpu as T  # noqa: E402


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(ROOT, "oracle", "_ref", "msda", "MultiScaleDeformableAttention.so")
    spec = importlib.util.spec_from_file_location("MultiScaleDeformableAttention", path)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    for case in T.REF_KERNEL_CASES:
        v, sh, ls, lo, w = T._dev(*T.make_case(*case, seed=21))
        arrs = {"out_f32": ref.ms_deform_attn_forward(v, sh, ls, lo, w, 64)}
        v64, lo64, w64 = v.double(), lo.double(), w.double()
        arrs["out_f64"] = ref.ms_deform_attn_forward(v64, sh, ls, lo64, w64, 64)
        go = torch.from_numpy(T.ref_kernel_grad_out(tuple(arrs["out_f64"].shape))).cuda()
        arrs["grad_value"], arrs["grad_loc"], arrs["grad_attw"] = ref.ms_deform_attn_backward(v64, sh, ls, lo64, w64, go, 64)
        stored = {}
        for k, t in arrs.items():
            stored[k] = T.ref_kernel_sample(t).cpu().numpy()
            stored[k + "_absmax"] = np.array(t.abs().max().item())
        name = f"msda_refkernel_{T.ref_kernel_id(case)}.npz"
        np.savez_compressed(os.path.join(out_dir, name), **stored)
        print("wrote", name, os.path.getsize(os.path.join(out_dir, name)))


if __name__ == "__main__":
    main()
