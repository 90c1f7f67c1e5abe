"""CPU: the GEMM epilogue never waits on a global load (cuobjdump of the built library, no GPU needed).

Bias, column scale and row mask reach shared memory by cp.async (LDGSTS) when a tile starts, and the residual by TMA,
so no gemm_bf16_wgmma_kernel instantiation may contain an LDG: a consumer thread that loads from global memory waits
one round trip for each load whose result it uses."""
import os
import re
import shutil
import subprocess

import pytest

from visionllm_b200 import _lib


def _gemm_sass():
    exe = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    out = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1) if "gemm_bf16_wgmma_kernel" in m.group(1) else None
            if cur:
                funcs[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]+\*/\s+\S", line):
            funcs[cur].append(line)
    assert funcs, "no gemm_bf16_wgmma_kernel in the library"
    return funcs


def test_no_global_load_in_any_gemm_instantiation():
    funcs = _gemm_sass()
    bad = {name: [l.strip() for l in lines if re.search(r"\bLDG(\.\w+)*\s", l)] for name, lines in funcs.items()}
    assert not any(bad.values()), {k: (len(v), v[:4]) for k, v in bad.items() if v}
