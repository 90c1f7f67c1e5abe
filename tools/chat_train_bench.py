"""One fwd+bwd multimodal chat training step on one H100 (visionllm_b200/train.py, B200VisionLLMv2ModelTrain).

    python tools/chat_train_bench.py [--rounds 3] [--iters 3] [--llm-layers 32] [--out FILE.json]

1. chat step: the pair_forward shape family -- InternViT-6B (frozen, 448 px, one tile per sample) -> pixel shuffle ->
   internvl_mlp -> Vicuna-7B (all 32 layers by default; `--llm-layers` cuts it) -- on a right-padded
   batch of two ragged sequences (lengths 1200 and 871 in 1200 positions, 256 image tokens each, an [EMB] block each).
   Reported: tokens/s over the valid tokens and over all positions, peak allocated memory.
2. decoder step at T % 256 == 0 (Vicuna-7B-shaped, 4 layers, 2 x 2048 tokens): without a mask and with an all-ones
   attention mask, alternated.  Both take the unmasked path; the two times should agree within the spread.  This shows
   that the mask check costs nothing within one build; it is not a comparison with an earlier build.

Every figure is the median over `--rounds` rounds of the median of `--iters` timed steps (CUDA events), with the spread
of the round medians.  The card's name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_bench import alternate, card  # noqa: E402

VICUNA = dict(hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_key_value_heads=32, vocab_size=32026,
              rms_norm_eps=1e-6, max_position_embeddings=4096)
IMP, EMB, DET, NE = 32000, 32010, 32020, 4


def _init(module):
    with torch.no_grad():
        for n, p in module.named_parameters():
            if p.dim() == 1 and "norm" in n:
                p.fill_(1.0)
            else:
                p.normal_(0.0, 0.02)


def chat_step_bench(rounds, iters, llm_layers):
    from transformers import LlamaConfig
    from visionllm_b200.internvit import B200InternVisionModel, InternVisionConfig
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.modeling import B200VisionLLMv2Model
    from visionllm_b200.train import B200VisionLLMv2ModelTrain
    torch.manual_seed(0)
    with torch.device("cuda"):
        vit = B200InternVisionModel(InternVisionConfig(image_size=448)).to(torch.bfloat16)
        llm = B200LlamaForCausalLM(LlamaConfig(num_hidden_layers=llm_layers, **VICUNA)).to(torch.bfloat16)
    cfg = SimpleNamespace(use_pixelshuffle=True, vl_bridge_type="internvl_mlp", vis_output_layer=-1, num_embs=NE,
                          imp_token_id=IMP, emb_token_id=EMB, det_tool_id=DET, seg_tool_id=-1, grd_tool_id=-1, pose_tool_id=-1)
    m = B200VisionLLMv2Model(cfg, vit, llm).to("cuda", torch.bfloat16)
    _init(m)
    m.freeze_vis_encoder()
    tr = B200VisionLLMv2ModelTrain(m)
    L, lens, n_img = 1200, [1200, 871], 256
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(1, 31000, (2, L), device="cuda", generator=g)
    ids[:, 10:10 + n_img] = IMP
    ids[:, 400] = DET
    ids[:, 401:401 + NE] = EMB + torch.arange(NE, device="cuda")
    mask = (torch.arange(L, device="cuda")[None] < torch.tensor(lens, device="cuda")[:, None]).long()
    ids[mask == 0] = 0
    labels = ids.clone()
    labels[:, :10 + n_img] = -100
    labels[mask == 0] = -100
    images = torch.randn(2, 3, 448, 448, device="cuda", generator=g).bfloat16()
    losses = []

    def step():
        for p in m.parameters():
            p.grad = None
        out = tr(input_ids=ids, attention_mask=mask, images=images, labels=labels.clone())
        out.loss.backward()
        losses.append(out.loss.detach())

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    res = alternate({"step": step}, rounds, iters, warmup=1)["step"]
    res["valid_tokens_per_s"] = sum(lens) / (res["median_ms"] * 1e-3)
    res["positions_per_s"] = 2 * L / (res["median_ms"] * 1e-3)
    res["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    res["loss_finite"] = bool(torch.isfinite(torch.stack(losses)).all())
    res["shape"] = dict(vit="InternViT-6B 448px frozen", bridge="internvl_mlp", llm=f"Vicuna-7B dims, {llm_layers} layers",
                        positions=L, lengths=lens, image_tokens=n_img)
    return res


def mask_path_bench(rounds, iters):
    from transformers import LlamaConfig
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    torch.manual_seed(0)
    with torch.device("cuda"):
        lm = B200LlamaForCausalLM(LlamaConfig(num_hidden_layers=4, **VICUNA)).to(torch.bfloat16)
    _init(lm)
    tr = B200LlamaForCausalLMTrain(lm)
    B, T = 2, 2048
    g = torch.Generator(device="cuda").manual_seed(2)
    emb = (torch.randn(B, T, 4096, device="cuda", generator=g) * 0.5).bfloat16()
    labels = torch.randint(0, 32026, (B, T), device="cuda", generator=g)
    ones = torch.ones(B, T, dtype=torch.long, device="cuda")

    def step(mask):
        for p in lm.parameters():
            p.grad = None
        loss, _, _ = tr(emb, labels, attention_mask=mask)
        loss.backward()

    res = alternate({"no_mask": lambda: step(None), "all_ones_mask": lambda: step(ones)}, rounds, iters)
    for r in res.values():
        r["tokens_per_s"] = B * T / (r["median_ms"] * 1e-3)
    res["shape"] = dict(layers=4, llm="Vicuna-7B dims", tokens=B * T)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--llm-layers", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("chat_train_bench.py measures on a GPU; none is visible")
    out = {"card_before": card()}
    out["decoder_step_mask_path"] = mask_path_bench(a.rounds, a.iters)
    torch.cuda.empty_cache()
    out["chat_step"] = chat_step_bench(a.rounds, a.iters, a.llm_layers)
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
