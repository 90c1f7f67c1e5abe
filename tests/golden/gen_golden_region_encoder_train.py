"""Golden vectors for region-encoder TRAINING from the REFERENCE's own `RegionEncoder('grid_sample')`
(visionllmv2/model/region_encoder.py:66-145) run forward and backward on CPU in this build container, in fp32 and in bf16.
The point draw (torch.multinomial, random by design) of the fp32 run is recorded and replayed for the bf16 run, and stored
so the B200 module can be fed the same points; the upstream gradient of the [regions, out_dim] output is seeded.  Every
parameter gradient is recorded: mask_embedding.{0,1,3,4,6}.* and up_dim.*."""
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from weights_util import key_shapes, seeded_state_dict  # noqa: E402

REF = "/root/reference/VisionLLMv2/visionllmv2/model/region_encoder.py"
CFG = dict(hidden_dim=64, embed_dim=256, out_dim=96, patch_size=14)


def main():
    spec = importlib.util.spec_from_file_location("ref_region_encoder", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = torch.Generator().manual_seed(5)
    B, Hh = 4, 112
    images = torch.randn(B, 3, Hh, Hh, generator=g).to(torch.bfloat16).float()
    masks = torch.zeros(B, 1, Hh, Hh)
    masks[0, 0, 10:70, 20:90] = 1                               # 4200 pixels: the 2304-point cap applies
    masks[1, 0, 50:, :40] = 1
    masks[2, 0, 5:8, 100:103] = 1                               # 9 points: fewer than one 16-point query group
    masks[3, 0, 30:60, 30:45] = 1
    masks[3, 0, 80:100, 60:110] = 1                             # two blobs
    feats = [(torch.randn(B, 64, 256, generator=g) * 0.5).to(torch.bfloat16).float() for _ in range(3)]
    gout = torch.randn(B, CFG["out_dim"], generator=g).to(torch.bfloat16).float()
    out = {"images": images.numpy(), "masks": masks.numpy(), "grad_out": gout.numpy(), "cfg": json.dumps(CFG)}
    for i, f in enumerate(feats):
        out[f"feat_{i}"] = f.numpy()
    torch.manual_seed(0)
    ref = mod.RegionEncoder(mask_pool_type="grid_sample", **CFG)
    ref.load_state_dict(seeded_state_dict(ref, 77))
    out["keys"] = json.dumps(key_shapes(ref))
    names = [n for n, _ in ref.named_parameters()]
    out["params"] = json.dumps(names)
    drawn = []
    real = mod.rand_sample

    def record(x, divisor, max_len):
        p = real(x, divisor, max_len)
        drawn.append(p.clone())
        return p
    mod.rand_sample = record
    o32 = ref(images, masks, feats)
    o32.backward(gout)
    g32 = {n: p.grad.detach().clone() for n, p in ref.named_parameters()}
    assert len(drawn) == len(feats) * B
    for i, p in enumerate(drawn):
        out[f"points_{i // B}_{i % B}"] = p.numpy()
    replay = iter(drawn)
    mod.rand_sample = lambda x, d, m: next(replay).to(x.dtype)
    ref.zero_grad()
    r16 = ref.to(torch.bfloat16)
    o16 = r16(images.to(torch.bfloat16), masks.to(torch.bfloat16), [f.to(torch.bfloat16) for f in feats])
    o16.backward(gout.to(torch.bfloat16))
    mod.rand_sample = real
    out["out_f32"], out["out_refbf16"] = o32.detach().numpy(), o16.detach().float().numpy()
    for n, p in r16.named_parameters():
        out[f"grad_f32/{n}"] = g32[n].numpy()
        out[f"grad_refbf16/{n}"] = p.grad.detach().float().numpy()
        print(n, tuple(p.shape), "bf16 rel_l2", float((p.grad.float() - g32[n]).norm() / g32[n].norm()))
    np.savez_compressed(os.path.join(HERE, "train_region_encoder.npz"), **out)


if __name__ == "__main__":
    main()
