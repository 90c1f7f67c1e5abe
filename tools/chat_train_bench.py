"""One fwd+bwd multimodal chat training step on one H100 (visionllm_b200/train.py, B200VisionLLMv2ModelTrain).

    python tools/chat_train_bench.py [--rounds 3] [--iters 3] [--llm-layers 32] [--regions K] [--out FILE.json]

1. chat step: the pair_forward shape family -- InternViT-6B (frozen, 448 px, one tile per sample) -> pixel shuffle ->
   internvl_mlp -> Vicuna-7B (all 32 layers by default; `--llm-layers` cuts it) -- on a right-padded
   batch of two ragged sequences (lengths 1200 and 871 in 1200 positions, 256 image tokens each, an [EMB] block each).
   Reported: tokens/s over the valid tokens and over all positions, peak allocated memory.
2. decoder step at T % 256 == 0 (Vicuna-7B-shaped, 4 layers, 2 x 2048 tokens): without a mask and with an all-ones
   attention mask, alternated.  Both take the unmasked path; the two times should agree within the spread.  This shows
   that the mask check costs nothing within one build; it is not a comparison with an earlier build.

3. with `--regions K`: a region encoder built as the reference builds it (hidden 256, embed = the ViT width 3200, out 4096,
   patch 14, 'grid_sample') and K <region> tokens per sample join the chat step.  Reported: the step with and without
   regions, alternated (fixed point draws, so the sampler is not in the step); the region encoder's own fwd+bwd
   (region_encoder_train); the same encoder as eager torch autograd in the reference's formulation on the same points
   (bf16 F.conv2d, the LayerNorm2d formula and F.gelu; the pooling, as the reference's point_sample call, one fp32
   F.grid_sample per level over all regions padded to the longest point list and masked); and the sampler (`rand_sample` per level and region, which synchronises with the
   host as the reference's does).

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


def eager_region_encoder(enc, images, masks, feats, pts):
    """The region encoder as eager torch autograd in the reference's formulation (region_encoder.py:98-145): the mask
    embedding in the parameters' dtype, the pooling in fp32 (`point_sample(masks_out.float(), ...)`) over the regions'
    point lists padded to the longest one, masked, summed and divided by the count, then cast back."""
    import torch.nn.functional as F
    me = enc.mask_embedding

    def ln2d(x, i):
        u = x.mean(1, keepdim=True)
        s = (x - u).pow(2).mean(1, keepdim=True)
        return me[i].weight[:, None, None] * ((x - u) / torch.sqrt(s + me[i].eps)) + me[i].bias[:, None, None]
    x = F.conv2d(torch.cat([images, masks.to(images.dtype)], 1), me[0].weight, me[0].bias, stride=me[0].stride)
    x = F.gelu(ln2d(x, 1))
    x = F.conv2d(x, me[3].weight, me[3].bias, stride=2)
    x = F.conv2d(F.gelu(ln2d(x, 4)), me[6].weight, me[6].bias)
    R, E, h, w = x.shape
    outs = []
    for lv, f in enumerate(feats):
        x = x + f.reshape(R, h, w, -1).permute(0, 3, 1, 2)
        p = torch.nn.utils.rnn.pad_sequence([q.float() for q in pts[lv]], batch_first=True, padding_value=-1)
        valid = (p.sum(-1) >= 0).float()                                            # [R, n]
        grid = (p[..., -2:].flip(-1) * 2 - 1).unsqueeze(2)                          # [R, n, 1, 2]
        s = F.grid_sample(x.float(), grid, align_corners=False)[..., 0]             # [R, E, n]
        pooled = ((s * valid[:, None]).sum(-1) / valid.sum(-1, keepdim=True)).nan_to_num().to(x.dtype)
        outs.append(enc.up_dim(pooled))
    return torch.stack(outs).mean(0)


def chat_step_bench(rounds, iters, llm_layers, n_regions=0):
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

    def step(input_ids=None, **kw):
        for p in m.parameters():
            p.grad = None
        out = tr(input_ids=ids if input_ids is None else input_ids, attention_mask=mask, images=images, labels=labels.clone(), **kw)
        out.loss.backward()
        losses.append(out.loss.detach())

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    if n_regions:
        return region_bench(m, tr, step, ids, images, labels, rounds, iters, n_regions, losses)
    res = alternate({"step": step}, rounds, iters, warmup=1)["step"]
    res["valid_tokens_per_s"] = sum(lens) / (res["median_ms"] * 1e-3)
    res["positions_per_s"] = 2 * L / (res["median_ms"] * 1e-3)
    res["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    res["loss_finite"] = bool(torch.isfinite(torch.stack(losses)).all())
    res["shape"] = dict(vit="InternViT-6B 448px frozen", bridge="internvl_mlp", llm=f"Vicuna-7B dims, {llm_layers} layers",
                        positions=L, lengths=lens, image_tokens=n_img)
    return res


def region_bench(m, tr, step, ids, images, labels, rounds, iters, K, losses):
    from visionllm_b200.modeling import region_encoder_inputs
    from visionllm_b200.region_encoder import B200RegionEncoder
    from visionllm_b200.train import region_encoder_train
    REG = 32021                                     # an unused id inside the vocabulary (IMP, EMB.., DET: 32000, 32010.., 32020)
    m.region_encoder = B200RegionEncoder(256, 3200, 4096, patch_size=14, mask_pool_type="grid_sample").to("cuda", torch.bfloat16)
    _init(m.region_encoder)
    m.use_region_encoder, m.reg_token_id = True, REG
    reg_ids = ids.clone()
    reg_ids[:, 300:300 + K] = REG
    g = torch.Generator(device="cuda").manual_seed(3)
    regions = []
    for b in range(2):
        r = torch.zeros(K, 448, 448, device="cuda", dtype=torch.bfloat16)
        for k in range(K):
            y0, x0 = (int(v) for v in torch.randint(0, 300, (2,), device="cuda", generator=g))
            r[k, y0:y0 + 40 + 25 * k, x0:x0 + 60 + 20 * k] = 1
        regions.append(r)
    with torch.no_grad():
        _, split_sizes, outs = m.vision_hidden_state(images)
    ri, rm, rf = region_encoder_inputs(images, regions, outs.hidden_states, split_sizes)
    enc = m.region_encoder
    pts = enc.draw_points(rm, 3)
    dout = torch.randn(2 * K, 4096, device="cuda", generator=g).bfloat16()

    def enc_ours():
        enc.zero_grad(set_to_none=True)
        region_encoder_train(enc, ri, rm, rf, sample_points=pts).backward(dout)

    def enc_eager():
        enc.zero_grad(set_to_none=True)
        eager_region_encoder(enc, ri, rm, rf, pts).backward(dout)

    res = alternate({"step": step, "step_regions": lambda: step(input_ids=reg_ids, regions=regions, region_sample_points=pts)},
                    rounds, iters, warmup=1)
    res.update(alternate({"region_encoder_fwd_bwd": enc_ours, "region_encoder_eager_torch": enc_eager}, rounds, iters,
                         warmup=1))
    res.update(alternate({"sampler_rand_sample": lambda: enc.draw_points(rm, 3)}, rounds, iters, warmup=1))
    res["loss_finite"] = bool(torch.isfinite(torch.stack(losses)).all())
    res["shape"] = dict(region_encoder="hidden 256, embed 3200, out 4096, patch 14, grid_sample", regions_per_sample=K,
                        points=[len(p) for p in pts[0]])
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
    ap.add_argument("--regions", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("chat_train_bench.py measures on a GPU; none is visible")
    out = {"card_before": card()}
    if a.regions:
        out["chat_step_regions"] = chat_step_bench(a.rounds, a.iters, a.llm_layers, a.regions)
    else:
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
