"""Golden vectors for the InternLM2 training wrapper on a right-padded, ragged batch (B200InternLM2ForCausalLMTrain with
`attention_mask`), produced by RUNNING THE REFERENCE'S OWN `InternLM2ForCausalLM` through torch autograd on CPU with the
same mask (build container only; needs the reference checkout; the reference builds its own 4-D causal + padding mask).
    python tests/golden/gen_golden_train_internlm2_padded.py

Shape and weights of train_internlm2_inputs.py, inputs of train_internlm2_padded_inputs.py (T = 200, lengths 200 / 101 /
13).  Two legs: fp32 and bf16 autograd; loss = CE over shifted labels on the fp32 logits, -100 at padded positions.
Stored as in gen_golden_train_internlm2.py: a seeded sample of flat indices per tensor and both legs' values there; the
logits are sampled at valid positions only (a padded position's logits are not part of the step).
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from train_internlm2_padded_inputs import B, CFG, T, WEIGHT_SEED, checksum, inputs  # noqa: E402
from weights_util import key_shapes, seeded_state_dict  # noqa: E402

torch.set_num_threads(8)

N_PARAM, N_BIG = 1024, 4096


def main():
    cfgm, mod = ref_shim.load_internlm2()
    cfg = cfgm.InternLM2Config(max_position_embeddings=256, attn_implementation="eager", bias=False, **CFG)
    cfg.rope_scaling = None          # transformers 5.x rewrites the field into a dict the 4.34-era code cannot read
    m = mod.InternLM2ForCausalLM(cfg)
    m.load_state_dict(seeded_state_dict(m, WEIGHT_SEED))
    emb, labels, mask = inputs()

    def run(dtype):
        mm = m.to(dtype).train(False)
        for p in mm.parameters():
            p.grad = None
        e = emb.clone().to(dtype).requires_grad_(True)
        out = mm(inputs_embeds=e, attention_mask=mask, use_cache=False, return_dict=True)
        logits = out.logits.float()
        loss = F.cross_entropy(logits[:, :-1].reshape(-1, CFG["vocab_size"]), labels[:, 1:].reshape(-1), ignore_index=-100)
        loss.backward()
        grads = {n: p.grad.detach().float().clone() for n, p in mm.named_parameters() if p.grad is not None}
        return float(loss), logits.detach(), e.grad.detach().float(), grads

    l32, lg32, de32, g32 = run(torch.float32)
    l16, lg16, de16, g16 = run(torch.bfloat16)
    sel = torch.Generator().manual_seed(6)
    arrs = dict(inputs_checksum=checksum(emb, labels).numpy(), mask=mask.numpy(), loss_f32=np.float64(l32),
                loss_refbf16=np.float64(l16))

    def sample(key, a32, a16, n, allowed=None):
        flat32, flat16 = a32.reshape(-1), a16.reshape(-1)
        pool = torch.arange(flat32.numel()) if allowed is None else allowed.reshape(-1).nonzero()[:, 0]
        idx = pool if pool.numel() <= n else pool[torch.randperm(pool.numel(), generator=sel)[:n]].sort().values
        arrs[key + "/idx"] = idx.to(torch.int32).numpy()
        arrs[key + "/f32"] = flat32[idx].numpy()
        arrs[key + "/refbf16"] = flat16[idx].numpy()

    sample("logits", lg32, lg16, N_BIG, mask.bool()[:, :, None].expand_as(lg32))
    sample("d_emb", de32, de16, N_BIG)
    for n in sorted(g32):
        sample("grad/" + n, g32[n], g16[n], N_PARAM)
    arrs["params"] = np.array(json.dumps(sorted(g32)))
    arrs["keys"] = np.array(json.dumps(key_shapes(m)))
    arrs["config"] = np.array(json.dumps(CFG))
    path = os.path.join(HERE, "train_internlm2_padded.npz")
    np.savez_compressed(path, **arrs)
    print("wrote", path, os.path.getsize(path), "bytes; loss", l32, l16, "params", len(g32),
          "d_emb at padded positions", float(de32[mask == 0].abs().max()))


if __name__ == "__main__":
    main()
