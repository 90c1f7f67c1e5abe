"""CPU: the SASS of every GEMM kernel instantiation (cuobjdump of the built library, no GPU needed).

- No HGMMA on a null descriptor (`gdesc[URZ]`): ptxas emits one when a `wgmma.commit_group` follows a branch that
  already closed the wgmma group, and the `wgmma.wait_group 1` after it then waits for the k-block just issued instead of
  the previous one -- every k-block drains the tensor pipe.  Keeping the k-block body one basic block (operand layouts
  as template parameters) prevents it.
- No local-memory loads or stores: the 64 / 128 fp32 accumulators per thread must stay in registers."""
import os
import re
import shutil
import subprocess

import pytest

from visionllm_b200 import _lib


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


@pytest.fixture(scope="module")
def gemm_sass():
    exe = _cuobjdump()
    if exe is None:
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


def test_every_instantiation_issues_hgmma(gemm_sass):
    for name, lines in gemm_sass.items():
        assert any("HGMMA" in l for l in lines), name


def test_no_hgmma_on_a_null_descriptor(gemm_sass):
    bad = {name: [l.strip() for l in lines if "HGMMA" in l and "gdesc[URZ]" in l] for name, lines in gemm_sass.items()}
    assert not any(bad.values()), {k: v for k, v in bad.items() if v}


def test_wait_follows_a_real_group(gemm_sass):
    # the instruction in front of every `DEPBAR.LE gsb0, 0x1` is the HGMMA that closes the k-block's group
    for name, lines in gemm_sass.items():
        for i, l in enumerate(lines):
            if re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", l):
                assert "HGMMA" in lines[i - 1] and "gsb0" in lines[i - 1], (name, lines[i - 1].strip(), l.strip())


def test_no_local_memory(gemm_sass):
    bad = {name: sum(1 for l in lines if re.search(r"\b(LDL|STL)(\.\w+)*\s", l)) for name, lines in gemm_sass.items()}
    assert not any(bad.values()), bad
