"""Golden vectors for tests/test_gdino_model_cpu.py: the REFERENCE's own `OVGroundingDinoForObjectDetection.forward_test`
on CPU in fp32 (needs a checkout of the reference project, see ref_shim.py) on the seeded weights and inputs that the test
rebuilds for itself.  Stored per case: the reference's state-dict keys / shapes and its outputs.

    python tests/golden/gen_golden_gdino_model_cpu.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ref_shim  # noqa: E402
import test_gdino_model_cpu as T  # noqa: E402
from weights_util import key_shapes  # noqa: E402


def reference(cfgm, gd, kw, seed):
    cfg = cfgm.GroundingDinoConfig(**kw)
    ref = gd.OVGroundingDinoForObjectDetection(cfg).eval()
    ref.load_state_dict(T.stage_state_dict(ref, seed))
    return ref


def outputs(ref, x, pm, tq, tm):
    with torch.no_grad():
        a = ref.forward_test(pixel_values=x, pixel_mask=pm, text_query=tq, text_query_masks=tm, return_dict=True)
    return dict(logits=a.logits.numpy(), pred_boxes=a.pred_boxes.numpy(), pred_masks=a.pred_masks.numpy())


def save(name, ref, arrs):
    path = os.path.join(HERE, name)
    np.savez_compressed(path, keys=np.array(json.dumps(key_shapes(ref))), **arrs)
    print("wrote", name, os.path.getsize(path))


def main():
    torch.set_num_threads(8)
    cfgm, gd = ref_shim.load_gdino()
    for ragged, b200_backbone in T.STAGE_CASES:
        ref = reference(cfgm, gd, dict(T.stage_kwargs(b200_backbone), disable_custom_kernels=True, fusion_dropout=0.,
                                       fusion_droppath=0., text_enhancer_dropout=0.), 11)
        save(T.stage_golden(ragged, b200_backbone), ref, outputs(ref, *T.stage_inputs(ragged)))
    ref = reference(cfgm, gd, dict(T.stage_kwargs(False), disable_custom_kernels=True, fusion_dropout=0., fusion_droppath=0.,
                                   text_enhancer_dropout=0.), 12)
    x, pm, tq, tm = T.neck_inputs()
    cap = {}
    orig = ref.model.encoder.forward

    def spy(**kw):
        cap.update(kw)
        return orig(**kw)

    ref.model.encoder.forward = spy
    with torch.no_grad():
        ref.forward_test(pixel_values=x, pixel_mask=pm, text_query=tq, text_query_masks=tm, return_dict=True)
    save("gdino_cpu_neck.npz", ref, {k: cap[k].numpy() for k in ("spatial_shapes", "level_start_index", "vision_attention_mask",
                                                                 "valid_ratios", "vision_features", "vision_position_embedding")})
    cfgm, gd = ref_shim.load_gdino_with_dcnv3()
    ref = reference(cfgm, gd, dict(T.internimage_kwargs(), disable_custom_kernels=True, fusion_dropout=0., fusion_droppath=0.,
                                   text_enhancer_dropout=0.), 21)
    save("gdino_cpu_internimage.npz", ref, outputs(ref, *T.internimage_inputs()))


if __name__ == "__main__":
    main()
