"""GPU: TFLOP/s of the wgmma GEMM (both tile widths) at the hot-path shapes; torch.matmul (cuBLAS) beside it.
Usage: python tools/gemm_bench.py [out.json]   (the card's name and power limit are recorded with the numbers)"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from visionllm_b200 import ops, _lib

SHAPES = {"vit_qkv": (41000, 9600, 3200), "vit_proj": (41000, 3200, 3200), "vit_fc1": (41000, 12800, 3200),
          "vit_fc2": (41000, 3200, 12800), "llm_qkv": (12288, 12288, 4096), "llm_gateup": (12288, 22016, 4096),
          "llm_down": (12288, 4096, 11008), "gdino_ffn1": (21760 * 8, 2048, 256), "sq8k": (8192, 8192, 8192)}
res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True).stdout.strip()}


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


for name, (M, N, K) in SHAPES.items():
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    fl = 2.0 * M * N * K
    r = {}
    for v, nm in ((1, "tile128x128"), (2, "tile128x256")):
        _lib.lib().vllm_gemm_set_variant(v)
        try:
            ms = timeit(lambda: ops.linear(x, w, out=out))
            r[f"{nm}_tflops"] = fl / ms / 1e9
        except Exception as e:
            r[f"{nm}_error"] = str(e)
    _lib.lib().vllm_gemm_set_variant(0)
    ms = timeit(lambda: torch.matmul(x, w.T, out=out))
    r["cublas_tflops"] = fl / ms / 1e9
    res[name] = r
    print(name, r, flush=True)
    del x, w, out
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"), indent=1)
