"""CPU: bench.py --dump-outputs -- which tensors of a step's result are stored, as what, and within which budget."""
import os
import subprocess
import sys
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench_workloads as B  # noqa: E402


def test_output_arrays_walks_nested_results_in_a_fixed_order():
    out = SimpleNamespace(logits=torch.zeros(2, 3), loss=None, past=(torch.ones(1), {"k": torch.ones(2), "n": 5}),
                          extra=OrderedDict(z=torch.zeros(1), a=[torch.zeros(4)]))
    names = [n for n, _ in B.output_arrays(out)]
    assert names == ["out.extra.z", "out.extra.a.0", "out.logits", "out.past.0", "out.past.1.k"]
    assert [n for n, _ in B.output_arrays(torch.zeros(3))] == ["out"]
    assert B.output_arrays(None) == [] and B.output_arrays(3.0) == []


def test_dump_outputs_types_budget_and_determinism(tmp_path):
    g = torch.Generator().manual_seed(1)
    big = torch.randn(300, 1000, generator=g)
    out = {"big": big, "half": torch.randn(5, 7, generator=g).bfloat16(), "idx": torch.arange(6).reshape(2, 3),
           "wide": torch.randn(4, generator=g).double(), "none": None}
    budget = 4 * 40000                                            # 4 tensors -> 40000 B each -> 10000 fp32 elements
    B.dump_outputs(out, str(tmp_path / "a"), budget_bytes=budget)
    B.dump_outputs(out, str(tmp_path / "b"), budget_bytes=budget)
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == ["out.big.npy", "out.half.npy", "out.idx.npy", "out.wide.npy"]
    a = {f: np.load(tmp_path / "a" / f) for f in files}
    assert all(np.array_equal(a[f], np.load(tmp_path / "b" / f)) for f in files)          # same positions every run
    assert a["out.half.npy"].dtype == np.float32 and a["out.half.npy"].shape == (5, 7)
    assert a["out.idx.npy"].dtype == np.float64 and a["out.idx.npy"].tolist() == [[0, 1, 2], [3, 4, 5]]
    assert a["out.wide.npy"].dtype == np.float64
    s = a["out.big.npy"]
    assert s.dtype == np.float32 and s.ndim == 1 and 5000 < s.size <= 10000
    flat = big.reshape(-1).numpy()
    step = -(-flat.size // 10000)
    assert any(np.array_equal(s, flat[o::step]) for o in range(step))                     # distinct, evenly spaced positions
    assert sum(os.path.getsize(tmp_path / "a" / f) for f in files) <= budget + 128 * len(files)
    assert B.DUMP_BUDGET_BYTES + 128 * 4096 <= 64 * 1000 * 1000                           # headers of thousands of files fit


def test_dump_outputs_is_refused_for_the_reference_arm(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "msda_encoder",
                        "--dump-outputs", str(tmp_path / "d")], capture_output=True, text=True)
    assert r.returncode != 0 and "--dump-outputs" in r.stderr and not (tmp_path / "d").exists()
