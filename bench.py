#!/usr/bin/env python
"""bench.py -- throughput of the VisionLLMv2 forward hot path.

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload NAME] [--dump-outputs DIR]

One JSON line on rank 0.  See DESIGN.md "Measurement" for what each field means.
Workloads live in bench_workloads.py; the default is the most complete
native path available (see DEFAULT_WORKLOAD there).  Nothing is written next to
the sources (no bytecode either), so the tree may be read-only; --dump-outputs
writes what the last timed step computed to DIR, for output-for-output
comparison of two builds (inputs and weights are seeded: same arguments, same
inputs).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


class ClockSampler:
    """nvidia-smi clocks/throttle reasons DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.proc, self.rows = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.index)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.12)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, pw = [], [], set(), []
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx.append(float(r[1])); pw.append(float(r[2]))
            except Exception:
                continue
            for name, col in (("hw_slowdown", 4), ("hw_thermal_slowdown", 5), ("sw_thermal_slowdown", 6),
                              ("sw_power_cap", 7)):
                if len(r) > col and r[col].lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(pw) if pw else None, "samples": len(sm), "reasons": sorted(reasons)}


_T0 = time.time()


def trace(msg):
    """Stage timestamps on stderr (VLLM_BENCH_TRACE=1): where a multi-rank launch spends its start-up time."""
    if os.environ.get("VLLM_BENCH_TRACE"):
        print(f"[bench rank {os.environ.get('RANK', '0')} +{time.time() - _T0:6.1f}s] {msg}", file=sys.stderr, flush=True)


_REAL_STDOUT = None


def quiet_stdout():
    """Libraries print to fd 1 (NCCL's "NCCL version ..." banner at communicator creation): park the real stdout and
    send everything else to stderr, so that the ONE JSON line is the only thing on stdout."""
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)


def emit(line):
    sys.stdout.flush()
    if _REAL_STDOUT is not None:
        os.dup2(_REAL_STDOUT, 1)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--workload", default=None)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy (float32 / float64, <= 64 MB in all; "
                         "larger arrays as a fixed seeded sample of their elements)")
    ap.add_argument("--cuprof", action="store_true",
                    help="wrap ONE extra device step in cudaProfilerStart/Stop (ncu --profile-from-start off)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "native" else max(args.warmup, 1)

    import bench_workloads as benchlib
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    name = args.workload or benchlib.DEFAULT_WORKLOAD

    if args.impl == "reference":
        if args.dump_outputs:
            ap.error("--dump-outputs stores the outputs of the native timed path; it has no meaning with --impl reference")
        # The reference's CPU implementation of the path, on the host cores; rank 0 only.
        if rank != 0:
            return
        line = benchlib.run_reference_arm(name, n_gpus=args.gpus, steps=args.steps, warmup=args.warmup)
        print(json.dumps(line), flush=True)
        return

    quiet_stdout()
    trace("importing torch")
    import torch
    import torch.distributed as dist
    trace("torch imported")
    torch.cuda.set_device(local_rank)
    torch.cuda.init()
    trace("cuda context up")
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        trace("process group up")
    wl = benchlib.WORKLOADS[name](rank=rank, world=world, device=torch.device("cuda", local_rank))
    wl.setup()
    trace("workload set up")

    from visionllm_b200 import _lib

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, warmup):
        """EXACTLY `steps` calls, barrier+sync on both sides, CUDA events, max over ranks -> ms total."""
        for _ in range(warmup):
            fn()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = _lib.launch_count()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        launches = _lib.launch_count() - l0
        barrier()
        return benchlib.max_over_ranks(e0.elapsed_time(e1), dist if world > 1 else None, "cuda"), launches

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ms_dev, launches = timed(wl.step_device, args.steps, args.warmup)
    trace(f"device-resident steps timed: {ms_dev / args.steps:.2f} ms/step")
    if args.dump_outputs and rank == 0:
        benchlib.dump_outputs(wl.out, args.dump_outputs)
    if args.cuprof:
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        wl.step_device()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
    kern = wl.dominant_kernel_ms(args.steps)            # live CUDA-event time of the dominant kernel
    ms_e2e, _ = timed(wl.step_e2e, args.steps, args.warmup)
    clocks = sampler.stop() if rank == 0 else None
    tp_obj = None
    if world > 1 and name == benchlib.DEFAULT_WORKLOAD and not os.environ.get("VLLM_BENCH_NO_EXTRAS"):
        try:                                               # cfg 5 under the same launch (all ranks take part)
            tp_obj = benchlib.tp_extra(rank, world, torch.device("cuda", local_rank))
        except Exception as e:
            tp_obj = {"error": f"{type(e).__name__}: {e}"[:300]}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    units = wl.units_per_step() * world
    peaks = benchlib.measured_peaks()
    roof = wl.roofline(kern, peaks)
    line = {
        "metric": wl.metric, "value": units / (ms_dev / args.steps / 1e3), "unit": wl.unit,
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_dev / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": wl.dtype,
        "data": "synthetic", "config": wl.config(),
        "e2e": {"value": units / (ms_e2e / args.steps / 1e3), "unit": wl.unit,
                "h2d_bytes_per_step": wl.h2d_bytes, "d2h_bytes_per_step": wl.d2h_bytes,
                "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": launches, "gpu": benchlib.gpu_identity(local_rank), "clocks": clocks, "roofline": roof,
        "max_memory_allocated_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
    }
    line["config"]["h100_80gb_peak_memory_gb"] = benchlib.H100_80GB_PEAK_GB.get(name)
    line.update(wl.extra())
    if tp_obj is not None:
        line["tp"] = tp_obj
    if name == benchlib.DEFAULT_WORKLOAD and not os.environ.get("VLLM_BENCH_NO_EXTRAS"):
        try:                                               # the "deform-attn HBM GB/s" half of BASELINE.json's metric
            line["msda"] = benchlib.msda_extra(torch.device("cuda", local_rank))
        except Exception as e:
            line["msda"] = {"error": f"{type(e).__name__}: {e}"[:300]}
    if not args.no_cpu_baseline and world == 1:
        line["cpu_baseline"] = benchlib.cpu_baseline(name)
    emit(line)
    if world > 1:
        os.dup2(2, 1)                                  # teardown chatter stays off stdout too
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
