"""GPU: fused attention TFLOP/s at the hot-path shapes, wgmma kernel vs warp-MMA kernel vs torch SDPA (library).
Usage: python tools/attn_bench.py [out.json]   (the card's name and power limit are recorded with the numbers)"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from visionllm_b200 import ops, _lib

SHAPES = {"vit_40x1025x25": (40, 1025, 25, False), "llm_8x1536x32_causal": (8, 1536, 32, True),
          "llm_2x3136x32_causal": (2, 3136, 32, True)}
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


for name, (B, T, H, causal) in SHAPES.items():
    qkv = torch.randn(B, T, 3, H, 128, device="cuda").bfloat16()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    fl = 4.0 * B * H * T * T * 128 * (0.5 if causal else 1.0)
    r = {}
    for var, nm in ((0, "wgmma"), (1, "warp_mma")):
        _lib.lib().vllm_attention_set_variant(var)
        try:
            ms = timeit(lambda: ops.attention(q, k, v, causal=causal))
            r[nm + "_tflops"] = fl / ms / 1e9
            r[nm + "_ms"] = ms
        except Exception as e:
            r[nm + "_error"] = str(e)
    _lib.lib().vllm_attention_set_variant(0)
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
    ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=causal))
    r["torch_sdpa_tflops"] = fl / ms / 1e9
    res[name] = r
    print(name, r, flush=True)
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"), indent=1)
