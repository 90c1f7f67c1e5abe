"""Build the REFERENCE's own MSDA CUDA extension (the kernel to beat, SURVEY 8c row 2 / BASELINE.md 4b) for sm_90.

Sources are taken where they lie in a checkout of the reference project (visionllmv2/model/unipose/ops/src -- the same
kernels as mmcv's ms_deform_attn_cuda_kernel.cuh; root = $VLLM_REFERENCE_ROOT, default: a directory `reference` next to
this repository), copied UNMODIFIED into oracle/_ref/msda/src (git-ignored, never committed), then three mechanical
API-compat edits are applied to the copies so that they compile against torch 2.11:
  * `#include <THC/THCAtomics.cuh>`  -> `#include <ATen/cuda/Atomic.cuh>`   (THC was removed from torch)
  * `x.type().is_cuda()`             -> `x.is_cuda()`
  * `AT_DISPATCH_FLOATING_TYPES(value.type(), ...)` -> `value.scalar_type()`; `.data<T>()` -> `.data_ptr<T>()`
No kernel arithmetic is touched.  Output: oracle/_ref/msda/MultiScaleDeformableAttention.so; tests/test_msda_gpu.py
compares our kernels with it and bench.py's `msda` object times it beside ours.  No GPU is needed to build (nvcc
cross-compiles); without the reference checkout nothing is built and those comparisons are skipped.

    python oracle/build_msda_ref.py
"""
import glob
import os
import re
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE_ROOT = os.environ.get("VLLM_REFERENCE_ROOT", os.path.join(os.path.dirname(ROOT), "reference"))
SRC = os.path.join(REFERENCE_ROOT, "VisionLLMv2", "visionllmv2", "model", "unipose", "ops", "src")
DST = os.path.join(ROOT, "oracle", "_ref", "msda")
NAME = "MultiScaleDeformableAttention"


def built_path():
    hits = glob.glob(os.path.join(DST, NAME + "*.so"))
    return hits[0] if hits else None


def main():
    if not os.path.isdir(SRC):
        print("reference sources not present: using the prebuilt", built_path())
        return 0 if built_path() else 1
    src = os.path.join(DST, "src")
    shutil.rmtree(src, ignore_errors=True)
    shutil.copytree(SRC, src)
    for path in glob.glob(os.path.join(src, "**", "*.*"), recursive=True):
        text = open(path).read()
        new = text.replace("#include <THC/THCAtomics.cuh>", "#include <ATen/cuda/Atomic.cuh>")
        new = new.replace(".type().is_cuda()", ".is_cuda()")
        new = re.sub(r"AT_DISPATCH_FLOATING_TYPES\((\w+)\.type\(\)", r"AT_DISPATCH_FLOATING_TYPES(\1.scalar_type()", new)
        new = re.sub(r"\.data<", ".data_ptr<", new)
        if new != text:
            open(path, "w").write(new)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils.cpp_extension import load
    build = os.path.join(DST, "build")
    os.makedirs(build, exist_ok=True)
    load(name=NAME, sources=[os.path.join(src, "vision.cpp"), os.path.join(src, "cpu", "ms_deform_attn_cpu.cpp"),
                             os.path.join(src, "cuda", "ms_deform_attn_cuda.cu")],
         extra_include_paths=[src], extra_cflags=["-DWITH_CUDA", "-O3"],
         extra_cuda_cflags=["-DWITH_CUDA", "-O3", "-lineinfo", "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__",
                            "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"],
         build_directory=build, is_python_module=False, verbose=True)
    so = glob.glob(os.path.join(build, NAME + "*.so"))[0]
    shutil.copy(so, os.path.join(DST, NAME + ".so"))
    print("built", os.path.join(DST, NAME + ".so"))
    return 0


if __name__ == "__main__":
    sys.exit(main())
