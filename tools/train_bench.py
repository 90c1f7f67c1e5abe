"""Training-side timings of grouped-query attention on one H100 (visionllm_b200/train.py).

    python tools/train_bench.py [--rounds 3] [--iters 5] [--skip-step] [--out FILE.json]

1. Attention backward at the InternLM2-20B layer shape (B 2, T 4096, 48 query heads over 8 KV heads, D 128), three
   variants alternated over `--rounds` rounds, each round the median of `--iters` timed calls (CUDA events):
     grouped   attention_backward_packed on the packed [B, T, G + 2, nkv, D] rows (grouped batched GEMMs)
     repeat    K / V repeated G times -> the same backward as MHA -> the G copies of dK / dV summed in fp32, rounded once
     sdpa      torch scaled_dot_product_attention (enable_gqa) backward on the same tensors
   Reported: the median over rounds and the spread (max - min) of the per-round medians.
2. One fwd+bwd step of a 4-layer InternLM2-20B-shaped decoder (H 6144, I 16384, V 92544, rope_theta 1e6) on 2 x 4096
   tokens through B200InternLM2ForCausalLMTrain: tokens/s (median and spread over rounds) and peak allocated memory.

The card's name, power limit and SM clocks are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return dict(zip(q.split(","), (s.strip() for s in r.stdout.strip().split(","))))
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def timed(fn, iters):
    """median ms per call over `iters` calls, each bracketed by CUDA events"""
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def alternate(variants, rounds, iters, warmup=2):
    for fn in variants.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    per = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            per[k].append(timed(fn, iters))
    return {k: {"median_ms": statistics.median(v), "spread_ms": max(v) - min(v), "rounds_ms": v} for k, v in per.items()}


def attention_backward_bench(rounds, iters):
    from visionllm_b200.train import attention_backward_packed
    B, T, nq, nkv, D = 2, 4096, 48, 8, 128
    G = nq // nkv
    scale = D ** -0.5
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv5 = (torch.randn(B, T, G + 2, nkv, D, device="cuda", generator=g) * 0.5).bfloat16()
    do = (torch.randn(B, T, nq * D, device="cuda", generator=g) * 0.5).bfloat16()

    def grouped():
        return attention_backward_packed(qkv5, do, scale)

    def repeat():
        q = qkv5[:, :, :G].reshape(B, T, nq, D)
        k = qkv5[:, :, G].repeat_interleave(G, 2)
        v = qkv5[:, :, G + 1].repeat_interleave(G, 2)
        d = attention_backward_packed(torch.stack((q, k, v), 2), do, scale)          # [B, T, 3, nq, D]
        dk = d[:, :, 1].view(B, T, nkv, G, D).float().sum(3).bfloat16()
        dv = d[:, :, 2].view(B, T, nkv, G, D).float().sum(3).bfloat16()
        return d[:, :, 0], dk, dv

    qt = qkv5[:, :, :G].reshape(B, T, nq, D).transpose(1, 2).detach().requires_grad_(True)
    kt = qkv5[:, :, G].transpose(1, 2).detach().requires_grad_(True)
    vt = qkv5[:, :, G + 1].transpose(1, 2).detach().requires_grad_(True)
    out = F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=scale, enable_gqa=True)
    dot = do.view(B, T, nq, D).transpose(1, 2)

    def sdpa():
        return torch.autograd.grad(out, (qt, kt, vt), dot, retain_graph=True)

    # the grouped and the repeat-then-sum gradients agree (both bf16 scores / probabilities; dK / dV rounded once)
    a, b = grouped(), repeat()
    dq_a, dk_a, dv_a = a[:, :, :G].reshape(B, T, nq, D), a[:, :, G], a[:, :, G + 1]
    agree = {n: float((x.float() - y.float()).norm() / y.float().norm())
             for n, x, y in (("dq", dq_a, b[0]), ("dk", dk_a, b[1]), ("dv", dv_a, b[2]))}
    del a, b
    torch.cuda.empty_cache()
    res = alternate({"grouped": grouped, "repeat": repeat, "sdpa": sdpa}, rounds, iters)
    flops = 2.0 * B * nq * T * T * D * 0.5 * 5                                      # 5 causal GEMMs of the backward
    for r in res.values():
        r["tflops_causal"] = flops / (r["median_ms"] * 1e-3) / 1e12
    return {"shape": dict(B=B, T=T, nq=nq, nkv=nkv, D=D), "rel_l2_grouped_vs_repeat": agree, "variants": res}


def step_bench(rounds, iters):
    from visionllm_b200.internlm2 import B200InternLM2ForCausalLM
    from visionllm_b200.train import B200InternLM2ForCausalLMTrain
    cfg = SimpleNamespace(vocab_size=92544, hidden_size=6144, intermediate_size=16384, num_hidden_layers=4,
                          num_attention_heads=48, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=1000000.0,
                          rope_scaling=None, hidden_act="silu", bias=False, pad_token_id=None)
    B, T = 2, 4096
    torch.manual_seed(0)
    with torch.device("cuda"):
        lm = B200InternLM2ForCausalLM(cfg).to(torch.bfloat16)
    with torch.no_grad():
        for n, p in lm.named_parameters():
            if "norm" in n:
                p.fill_(1.0)
            else:
                p.normal_(0.0, 0.02)
    tr = B200InternLM2ForCausalLMTrain(lm)
    g = torch.Generator(device="cuda").manual_seed(1)
    emb = (torch.randn(B, T, cfg.hidden_size, device="cuda", generator=g) * 0.5).bfloat16()
    labels = torch.randint(0, cfg.vocab_size, (B, T), device="cuda", generator=g)
    labels[:, :256] = -100
    losses = []

    def step():
        for p in lm.parameters():
            p.grad = None
        loss, _, _ = tr(emb, labels)
        loss.backward()
        losses.append(loss.detach())

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    res = alternate({"step": step}, rounds, iters, warmup=1)["step"]
    res["tokens_per_s"] = B * T / (res["median_ms"] * 1e-3)
    res["tokens_per_s_range"] = [B * T / (max(res["rounds_ms"]) * 1e-3), B * T / (min(res["rounds_ms"]) * 1e-3)]
    res["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    res["loss_finite"] = bool(torch.isfinite(torch.stack(losses)).all())
    res["shape"] = dict(layers=4, H=6144, I=16384, V=92544, nq=48, nkv=8, tokens=B * T)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_bench.py measures on a GPU; none is visible")
    out = {"card_before": card()}
    out["attention_backward"] = attention_backward_bench(a.rounds, a.iters)
    torch.cuda.empty_cache()
    if not a.skip_step:
        out["internlm2_4layer_step"] = step_bench(a.rounds, max(1, a.iters // 2))
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
