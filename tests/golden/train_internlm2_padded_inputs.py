"""Right-padded, ragged inputs of tests/golden/train_internlm2_padded.npz, shared by its generator and the tests that read
it: the shape and weights of train_internlm2_inputs.py at T = 200 (not a multiple of 256), three rows of lengths
200 / 101 / 13 (attention_mask 1 on the first `len` positions), labels -100 at the padded positions and on a prefix."""
import torch

from train_internlm2_inputs import CFG, WEIGHT_SEED, checksum  # noqa: F401

B, T = 3, 200
LENS = (200, 101, 13)


def inputs():
    """(inputs_embeds fp32 [B, T, H] with bf16-representable values, labels int64 [B, T], attention_mask int64 [B, T])"""
    g = torch.Generator().manual_seed(12)
    emb = (torch.randn(B, T, CFG["hidden_size"], generator=g) * 0.5).bfloat16().float()
    labels = torch.randint(0, CFG["vocab_size"], (B, T), generator=g)
    mask = (torch.arange(T)[None] < torch.tensor(LENS)[:, None]).long()
    labels[:, :5] = -100
    labels[mask == 0] = -100
    return emb, labels, mask
