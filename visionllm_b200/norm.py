"""Drop-in for the reference's third operator boundary: apex `FusedRMSNorm` (SURVEY 8b, boundary 3).

The reference swaps its RMSNorm implementation by REBINDING A MODULE ATTRIBUTE:
  * visionllmv2/train/llama_forward_monkey_patch.py:168-180  `replace_llama_rmsnorm_with_fused_rmsnorm()` sets
    `transformers.models.llama.modeling_llama.LlamaRMSNorm = partial(FusedRMSNorm, eps=1e-6)`;
  * visionllmv2/model/internvit/modeling_intern_vit.py:47-58  tries `from apex.normalization import FusedRMSNorm` and
    rebinds `InternRMSNorm` to it.
`B200RMSNorm` has FusedRMSNorm's constructor (`normalized_shape, eps, elementwise_affine`) and parameter name (`weight`),
its forward is `vllm_rmsnorm_bf16` (fp32 statistics, x * rsqrt rounded to the input dtype THEN times weight -- the
semantics of apex `cuApplyRMSNorm` / `manual_rms_norm`, apex/normalization/fused_layer_norm.py:16-29), and it is
differentiable through `train.RMSNormFn`, whose backward is `vllm_rmsnorm_bwd_ws_bf16` (apex `rms_backward_affine`;
the weight gradient summed in a fixed order, so it is deterministic).  `install()` performs the same rebinding.
"""
import numbers

import torch
import torch.nn as nn


class B200RMSNorm(nn.Module):
    def __init__(self, normalized_shape, eps=1e-5, elementwise_affine=True, **unused):
        super().__init__()
        if isinstance(normalized_shape, numbers.Integral):
            normalized_shape = (int(normalized_shape),)
        self.normalized_shape = torch.Size(normalized_shape)
        if len(self.normalized_shape) != 1:
            raise NotImplementedError("B200RMSNorm: one normalised dimension (the hidden size), as on the reference's path")
        self.eps = eps
        self.variance_epsilon = eps                     # HF LlamaRMSNorm's attribute name
        self.elementwise_affine = elementwise_affine
        if elementwise_affine:
            self.weight = nn.Parameter(torch.ones(self.normalized_shape))
        else:
            self.register_buffer("weight", torch.ones(self.normalized_shape), persistent=False)

    def forward(self, x):
        from . import ops
        from .train import RMSNormFn
        xc = x if x.is_contiguous() else x.contiguous()
        w = self.weight if self.weight.dtype == xc.dtype else self.weight.to(xc.dtype)
        if torch.is_grad_enabled() and (xc.requires_grad or w.requires_grad):
            return RMSNormFn.apply(xc, w, self.eps)
        return ops.rmsnorm(xc, w, self.eps)

    def extra_repr(self):
        return f"{tuple(self.normalized_shape)}, eps={self.eps}, elementwise_affine={self.elementwise_affine}"


def install(llama=True, internvit_module=None, internlm2_module=None):
    """The reference's own injection mechanism: rebind the RMSNorm class where its model files look it up.
    Call BEFORE the models are constructed (as the reference calls replace_llama_rmsnorm_with_fused_rmsnorm() first)."""
    from functools import partial
    done = []
    if llama:
        import transformers.models.llama.modeling_llama as ml
        ml.LlamaRMSNorm = partial(B200RMSNorm, eps=1e-6)       # llama_forward_monkey_patch.py:172-173 (HF passes eps= explicitly)
        done.append("transformers.models.llama.modeling_llama.LlamaRMSNorm")
    if internvit_module is not None:                           # modeling_intern_vit.py:47-58
        internvit_module.InternRMSNorm = B200RMSNorm
        done.append(internvit_module.__name__ + ".InternRMSNorm")
    if internlm2_module is not None:                           # internlm2/modeling_internlm2.py:114-128
        internlm2_module.InternLM2RMSNorm = B200RMSNorm
        done.append(internlm2_module.__name__ + ".InternLM2RMSNorm")
    return done
