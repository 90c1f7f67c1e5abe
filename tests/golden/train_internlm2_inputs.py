"""Shape and seeded inputs of tests/golden/train_internlm2_small.npz, shared by its generator and the tests that read it
(inputs and weights are regenerated from seeds, not stored; the golden keeps a checksum of the inputs so a change in
torch's CPU generator fails loudly instead of comparing against other numbers)."""
import torch

CFG = dict(vocab_size=1000, hidden_size=768, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=12,
           num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=1000000.0)
B, T = 2, 256
WEIGHT_SEED = 707


def inputs():
    """(inputs_embeds fp32 [B, T, H] with bf16-representable values, labels int64 [B, T] with a -100 prefix)"""
    g = torch.Generator().manual_seed(11)
    emb = (torch.randn(B, T, CFG["hidden_size"], generator=g) * 0.5).bfloat16().float()
    labels = torch.randint(0, CFG["vocab_size"], (B, T), generator=g)
    labels[:, :100] = -100                                           # visual positions carry no language loss
    return emb, labels


def checksum(emb, labels):
    """float64 [3]: sum, sum of squares of the inputs and the sum of the labels"""
    e = emb.double()
    return torch.tensor([float(e.sum()), float((e * e).sum()), float(labels.double().sum())], dtype=torch.float64)
