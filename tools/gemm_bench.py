"""GPU: TFLOP/s of the wgmma GEMM (both tile widths, forced) at the hot-path shapes, each with the epilogue it runs in the model;
torch.matmul (cuBLAS, no epilogue) beside it.  The three arms alternate, REPEATS rounds of each; the median and the spread
(max - min over the rounds) are printed.  The card's name, power limit and clocks are read in the same call.
Usage: python tools/gemm_bench.py [out.json] [shape ...]
       python tools/gemm_bench.py --ksweep [out.json]

--ksweep times one M x N shape at several K for each tile width and each epilogue kind and fits t = a + b*K by least
squares: a is the fixed cost of the launch's tiles (prologue, epilogue, pipeline fill), reported per tile as a / (tiles
per CTA), and 2*M*N / b is the main-loop rate.  M = 132 * 128 and N = 4096 give whole waves on a 132-SM H100 at both
tile widths, so every CTA runs the same number of tiles."""
import json, os, statistics, subprocess, sys
import numpy
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from visionllm_b200 import ops, _lib

# name: (M, N, K, epilogue); epilogue keys: bias, act, ls (column scale), res (residual), f32 (fp32 output)
SHAPES = {
    "vit_qkv": (41000, 9600, 3200, dict(bias=True)),
    "vit_proj": (41000, 3200, 3200, dict(bias=True, ls=True, res=True)),
    "vit_fc1": (41000, 12800, 3200, dict(bias=True, act="gelu")),
    "vit_fc2": (41000, 3200, 12800, dict(bias=True, ls=True, res=True)),
    "llm_qkv": (12288, 12288, 4096, dict()),
    "llm_o": (12288, 4096, 4096, dict(res=True)),
    "llm_gateup": (12288, 22016, 4096, dict(act="swiglu")),
    "llm_down": (12288, 4096, 11008, dict(res=True)),
    "lm_head": (12288, 32026, 4096, dict(f32=True)),
    "gdino_ffn1": (21760 * 8, 2048, 256, dict(bias=True, act="relu")),
    "sq8k": (8192, 8192, 8192, dict()),
}
REPEATS = 3
ARMS = (("tile128x128", _lib.GEMM_NARROW_TILE), ("tile128x256", _lib.GEMM_WIDE_TILE), ("cublas", None))


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


def timeit(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_shape(M, N, K, epi, arms=ARMS):
    dev = "cuda"
    x = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).bfloat16()
    act = epi.get("act")
    n_out = N // 2 if act == "swiglu" else N
    bias = torch.randn(N, device=dev).bfloat16() if epi.get("bias") else None
    ls = torch.rand(N, device=dev).bfloat16() if epi.get("ls") else None
    res = torch.randn(M, n_out, device=dev).bfloat16() if epi.get("res") else None
    if epi.get("f32"):
        out = torch.empty(M, (N + 7) // 8 * 8, device=dev, dtype=torch.float32)[:, :N]     # 16-byte row pitch, like the LLM logits
    else:
        out = torch.empty(M, n_out, device=dev, dtype=torch.bfloat16)
    cb_out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ours = lambda: ops.linear(x, w, bias=bias, act=act, colscale=ls, residual=res, out=out)
    cublas = lambda: torch.matmul(x, w.T, out=cb_out)
    iters = max(3, min(20, int(2e13 / (2.0 * M * N * K))))       # about 40 ms of work per timing at ~500 TFLOP/s
    times = {nm: [] for nm, _ in arms}
    for nm, v in arms:                                           # warm every arm (module load, cuBLAS heuristics)
        with _lib.knob("gemm_set_variant", v if v is not None else _lib.GEMM_DEFAULT):
            (cublas if v is None else ours)()
    torch.cuda.synchronize()
    for _ in range(REPEATS):
        for nm, v in arms:
            if v is None:
                times[nm].append(timeit(cublas, iters))
            else:
                with _lib.knob("gemm_set_variant", v):
                    times[nm].append(timeit(ours, iters))
    fl = 2.0 * M * N * K
    r = {}
    for nm, ts in times.items():
        tf = [fl / t / 1e9 for t in ts]
        r[nm] = {"tflops_median": statistics.median(tf), "tflops_spread": max(tf) - min(tf), "ms_median": statistics.median(ts)}
    return r


KSWEEP_M, KSWEEP_N, KSWEEP_K = 132 * 128, 4096, (256, 512, 1024, 2048, 3200)
KSWEEP_EPIS = {"none": dict(), "bias": dict(bias=True), "bias_ls_res": dict(bias=True, ls=True, res=True),
               "gelu": dict(bias=True, act="gelu"), "swiglu": dict(act="swiglu"), "f32": dict(f32=True)}


def ksweep():
    M, N = KSWEEP_M, KSWEEP_N
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {}
    for epi_name, epi in KSWEEP_EPIS.items():
        ts = {nm: [] for nm, _ in ARMS[:2]}
        for K in KSWEEP_K:
            r = bench_shape(M, N, K, epi, arms=ARMS[:2])
            for nm in ts:
                ts[nm].append(r[nm]["ms_median"])
            torch.cuda.empty_cache()
        for nm, t in ts.items():
            bn = 128 if nm == "tile128x128" else 256
            tiles = -(-M // 128) * -(-N // bn)
            b, a = numpy.polyfit(KSWEEP_K, t, 1)                 # t [ms] = a + b * K
            fit = [a + b * k for k in KSWEEP_K]
            res[f"{epi_name}/{nm}"] = {"ms": t, "a_ms": a, "a_us_per_tile": a * 1e3 / (tiles / min(sms, tiles)),
                                       "mainloop_tflops": 2.0 * M * N / b / 1e9,
                                       "max_fit_residual_us": max(abs(x - y) for x, y in zip(t, fit)) * 1e3}
            v = res[f"{epi_name}/{nm}"]
            print(f"{epi_name:12s} {nm}: fixed {v['a_us_per_tile']:.2f} us/tile, main loop {v['mainloop_tflops']:.0f} "
                  f"TFLOP/s, fit residual <= {v['max_fit_residual_us']:.1f} us; ms at K={list(KSWEEP_K)}: "
                  + " ".join(f"{x:.3f}" for x in t), flush=True)
    return res


def main():
    args = sys.argv[1:]
    sweep = "--ksweep" in args
    args = [a for a in args if a != "--ksweep"]
    out_path = args.pop(0) if args and args[0].endswith(".json") else None
    if sweep:
        res = {"gpu_before": gpu_state(), "shape_MN": [KSWEEP_M, KSWEEP_N]}
        print("gpu (name, power limit, SM clock, max SM clock, throttle reasons):", res["gpu_before"], flush=True)
        res["ksweep"] = ksweep()
        res["gpu_after"] = gpu_state()
        print("gpu after:", res["gpu_after"], flush=True)
        if out_path:
            with open(out_path, "w") as f:
                json.dump(res, f, indent=1)
        return
    names = args or list(SHAPES)
    res = {"gpu_before": gpu_state()}
    print("gpu (name, power limit, SM clock, max SM clock, throttle reasons):", res["gpu_before"], flush=True)
    for name in names:
        M, N, K, epi = SHAPES[name]
        r = bench_shape(M, N, K, epi)
        r["shape"] = [M, N, K]; r["epilogue"] = epi
        res[name] = r
        print(f"{name:11s} {M}x{N}x{K} {epi}: " +
              "  ".join(f"{nm} {v['tflops_median']:.0f}±{v['tflops_spread']:.0f}" for nm, v in r.items() if isinstance(v, dict)
                        and "tflops_median" in v), flush=True)
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_state()
    print("gpu after:", res["gpu_after"], flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
