"""Training-side path of the LLM decoder (BASELINE cfg 5: "fwd+bwd step", loss = CE on the text positions).

The reference trains `VisionLLMv2Model` through torch autograd over HF `LlamaForCausalLM` (third-party transformers) and
computes the language loss at visionllmv2/model/modeling_visionllmv2.py:741-757 (shift by one, CrossEntropyLoss, -100 =
IGNORE_INDEX; labels of the [EMB] slots are ignored).  Here every op of the decoder layer is a `torch.autograd.Function`
whose forward AND backward are this repo's kernels:

  op                forward                                   backward
  Linear            wgmma GEMM (ops.linear)                 dgrad / wgrad on the same kernel with MN-major operands
                                                              (ops.gemm_tn: no transposed copies of W, dy or x)
  RMSNorm           vllm_rmsnorm_bf16                         vllm_rmsnorm_bwd_ws_bf16 (dx + fp32 dweight, summed in
                                                              a fixed order through per-CTA partials)
  RoPE              vllm_rope_bf16 (q and k heads)            the same kernel with -sin (the rotation's transpose)
  causal attention  wgmma flash forward (ops.attention)     materialised backward: 5 block-diagonal batched wgmma GEMMs
                                                              over all (batch, head) matrices of the layer with causal
                                                              tile / K-range skipping + two row kernels (softmax recompute,
                                                              softmax backward); scores / probabilities in bf16 like HF's
                                                              eager bf16 attention; grouped-query attention reads KV
                                                              matrix i / G and reduces dK / dV over the G query
                                                              matrices of a KV head inside the GEMM (no repeated K / V)
  SwiGLU            vllm_swiglu_fwd_bf16 on the gate|up GEMM  vllm_swiglu_bwd_bf16
  CE loss           vllm_ce_loss_f32 (loss + dlogits in one pass over the fp32 logits); the upstream gradient
                                                              scales dlogits in place (vllm_scale_rows_bf16)

`B200LlamaForCausalLMTrain` / `B200InternLM2ForCausalLMTrain` wrap the inference module's parameters (same state dict)
and run a fwd+bwd step; both share one per-layer loop (`decoder_layer_train`).
Out of scope here (stated): the optimizer, gradient accumulation across micro-batches, the tensor-parallel exchange of
the backward (tp.py is forward-only) -- multi-GPU runs of this path are data-parallel replicas.
"""
import torch
import torch.nn as nn

from . import _lib, ops
from .llama import rope_tables


# ---- thin wrappers over the C-ABI row kernels ------------------------------------------------------------------------
def rmsnorm_bwd(x2, weight, dy2, eps):
    rows, cols = x2.shape
    dx = torch.empty_like(x2)
    dw = torch.empty(cols, dtype=torch.float32, device=x2.device)
    L = _lib.lib()
    n_part = L.vllm_rmsnorm_bwd_partials(rows)
    part = torch.empty((n_part, cols), dtype=torch.float32, device=x2.device)     # per-CTA dweight partials, summed in order
    with torch.cuda.device(x2.device):
        rc = L.vllm_rmsnorm_bwd_ws_bf16(x2.data_ptr(), x2.stride(0), weight.data_ptr(), dy2.data_ptr(), dy2.stride(0),
                                        dx.data_ptr(), dx.stride(0), dw.data_ptr(), part.data_ptr(), n_part, rows, cols,
                                        float(eps), ops._stream())
    _lib.check(rc, "vllm_rmsnorm_bwd_ws_bf16")
    return dx, dw


def swiglu_fwd(gu):
    rows, two_i = gu.shape
    h = torch.empty((rows, two_i // 2), dtype=gu.dtype, device=gu.device)
    with torch.cuda.device(gu.device):
        rc = _lib.lib().vllm_swiglu_fwd_bf16(gu.data_ptr(), gu.stride(0), h.data_ptr(), h.stride(0), rows, two_i // 2, ops._stream())
    _lib.check(rc, "vllm_swiglu_fwd_bf16")
    return h


def swiglu_bwd(gu, dh):
    rows, two_i = gu.shape
    dgu = torch.empty_like(gu)
    with torch.cuda.device(gu.device):
        rc = _lib.lib().vllm_swiglu_bwd_bf16(gu.data_ptr(), gu.stride(0), dh.data_ptr(), dh.stride(0), dgu.data_ptr(),
                                             dgu.stride(0), rows, two_i // 2, ops._stream())
    _lib.check(rc, "vllm_swiglu_bwd_bf16")
    return dgu


def head_stack(t, B, T, parts, H, D, to_stacked):
    """[B, T, parts, H, D] -> [parts, B, H, T, D] (to_stacked) or back, one 16-byte-vector pass (vllm_head_stack_bf16)."""
    src = t if t.is_contiguous() else t.contiguous()
    out = torch.empty((parts, B, H, T, D) if to_stacked else (B, T, parts, H, D), dtype=src.dtype, device=src.device)
    with torch.cuda.device(src.device):
        rc = _lib.lib().vllm_head_stack_bf16(src.data_ptr(), out.data_ptr(), B, T, parts, H, D, 1 if to_stacked else 0, ops._stream())
    _lib.check(rc, "vllm_head_stack_bf16")
    return out


def head_stack_qkv(qkv, nq, nkv, D, stacks=None):
    """Packed projection rows qkv [B, T, >= (nq + 2 nkv) D] (row pitch qkv.stride(1), q | k | v heads) -> one buffer
    [(nq + 2 nkv) B T, D] holding the stacks Q [B, nq, T, D] | K [B, nkv, T, D] | V [B, nkv, T, D]
    (vllm_head_stack_qkv_bf16).  With `stacks` given, the inverse: the stacks are written back into qkv."""
    B, T = qkv.shape[0], qkv.shape[1]
    to_stacked = stacks is None
    if to_stacked:
        stacks = torch.empty(((nq + 2 * nkv) * B * T, D), dtype=qkv.dtype, device=qkv.device)
    nq_rows, nkv_rows = B * nq * T, B * nkv * T
    q, k, v = stacks[:nq_rows], stacks[nq_rows:nq_rows + nkv_rows], stacks[nq_rows + nkv_rows:]
    with torch.cuda.device(qkv.device):
        rc = _lib.lib().vllm_head_stack_qkv_bf16(qkv.data_ptr(), qkv.stride(1), q.data_ptr(), k.data_ptr(), v.data_ptr(), B, T,
                                                 nq, nkv, D, 1 if to_stacked else 0, ops._stream())
    _lib.check(rc, "vllm_head_stack_qkv_bf16")
    return stacks if to_stacked else qkv


def gemm_batched(a, b, n_batch, M, N, K, a_mn=False, b_mn=False, causal=0, out_dtype=torch.bfloat16, out=None, group=1,
                 reduce=False):
    """Block-diagonal products in one wgmma launch (operands / output stacked along rows; vllm_gemm_bf16_batched_grouped):
    n_batch products C_i = A_i . B_{i // group}^T, or with `reduce` the n_batch // group sums over g < group of
    A_{j group + g} . B_{j group + g}^T."""
    if out is None:
        out = torch.empty(((n_batch // group if reduce else n_batch) * M, N), dtype=out_dtype, device=a.device)
    with torch.cuda.device(a.device), ops._Prof("gemm", 2.0 * n_batch * M * N * K * (0.5 if causal else 1.0), 0.0,
                                               f"b{n_batch}x{M}x{N}x{K}" + (f"g{group}{'r' if reduce else ''}" if group > 1 else "")):
        rc = _lib.lib().vllm_gemm_bf16_batched_grouped(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
                                                       out.data_ptr(), out.stride(0), n_batch, group, int(reduce), M, N, K,
                                                       int(causal), 1 if out_dtype == torch.float32 else 0, ops._stream())
    _lib.check(rc, "vllm_gemm_bf16_batched_grouped")
    return out


def attention_backward_packed(qkv5, do, scale):
    """Backward of causal softmax(q k^T * scale) v for the PACKED projection output qkv5 [B, T, G + 2, nkv, D] (bf16: the
    nq = G * nkv query heads, then the nkv key heads, then the nkv value heads of a row; q head i attends with KV head
    i // G, as HF's repeat_kv; MHA is G = 1, [B, T, 3, H, D]) and do [B, T, nq*D].  Returns d(qkv5) in the same packed
    layout.  The (batch, head) matrices are stacked along rows for the block-diagonal batched GEMMs by ONE copy of qkv5
    (and one of do); the three gradient GEMMs write one stacked buffer that ONE copy turns back into the packed layout.
    Grouped-query attention needs no repeated K / V: S, dP and dQ read KV matrix i // G, and dK, dV reduce over the G
    query matrices of a KV head inside one GEMM (fp32 accumulation, one rounding)."""
    B, T, parts, nkv, D = qkv5.shape
    G = parts - 2
    if G < 1 or T % 256 or D % 64:
        raise RuntimeError("attention_backward: sequence length must be a multiple of 256 and head_dim of 64")
    nq = G * nkv
    BQ, BKV = B * nq, B * nkv
    rows = qkv5.reshape(B, T, -1)                                               # a view for the decoder's packed projection
    if rows.stride(2) != 1 or rows.stride(1) % 8 or rows.data_ptr() % 16:
        rows = rows.contiguous()
    stk = head_stack_qkv(rows, nq, nkv, D)                                      # Q | K | V stacks, [(b, h), T, D] each
    qs, ks, vs = stk[:BQ * T], stk[BQ * T:(BQ + BKV) * T], stk[(BQ + BKV) * T:]
    dos = head_stack(do, B, T, 1, nq, D, True).view(BQ * T, D)
    L_ = _lib.lib()
    p = gemm_batched(qs, ks, BQ, T, T, D, causal=1, group=G)                     # S = Q K^T, tiles above the diagonal skipped
    with torch.cuda.device(qkv5.device):
        _lib.check(L_.vllm_softmax_causal_bf16(p.data_ptr(), p.stride(0), BQ, T, float(scale), ops._stream()), "vllm_softmax_causal_bf16")
    dp = gemm_batched(dos, vs, BQ, T, T, D, causal=1, group=G)                   # dP = dO V^T
    with torch.cuda.device(qkv5.device):
        _lib.check(L_.vllm_attn_ds_bf16(p.data_ptr(), dp.data_ptr(), p.stride(0), BQ, T, float(scale), ops._stream()), "vllm_attn_ds_bf16")
    ds = dp
    dstk = torch.empty_like(stk)
    dqs, dks, dvs = dstk[:BQ * T], dstk[BQ * T:(BQ + BKV) * T], dstk[(BQ + BKV) * T:]
    gemm_batched(p, dos, BQ, T, D, T, a_mn=True, b_mn=True, causal=2, out=dvs, group=G, reduce=True)   # dV = sum_g P_g^T dO_g
    gemm_batched(ds, qs, BQ, T, D, T, a_mn=True, b_mn=True, causal=2, out=dks, group=G, reduce=True)   # dK = sum_g dS_g^T Q_g
    gemm_batched(ds, ks, BQ, T, D, T, b_mn=True, causal=3, out=dqs, group=G)                            # dQ = dS K
    dqkv = torch.empty((B, T, parts * nkv * D), dtype=qkv5.dtype, device=qkv5.device)
    return head_stack_qkv(dqkv, nq, nkv, D, stacks=dstk).view(B, T, parts, nkv, D)  # packed gradient


def attention_backward(q, k, v, do, scale):
    """Backward for separate q [B, T, nq, D], k, v [B, T, nkv, D], do [B, T, nq, D].  Returns (dq, dk, dv) in the same
    layouts."""
    B, T, nq, D = q.shape
    nkv = k.shape[2]
    G = nq // nkv
    d = attention_backward_packed(torch.cat((q, k, v), 2).view(B, T, G + 2, nkv, D), do.reshape(B, T, -1), scale)
    return d[:, :, :G].flatten(2, 3), d[:, :, G], d[:, :, G + 1]


# ---- autograd Functions --------------------------------------------------------------------------------------------------
class LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, out_f32=False, residual=None):
        ctx.save_for_backward(x, weight)
        ctx.has_res = residual is not None
        if not out_f32:
            return ops.linear(x, weight, residual=residual)      # y = x W^T (+ residual in the GEMM epilogue)
        assert residual is None
        # fp32 rows need a 16-byte pitch (V = 32026 is not a multiple of 4): pad the pitch, return the [.., :V] view
        N = weight.shape[0]
        rows = x.numel() // x.shape[-1]
        buf = torch.empty((rows, (N + 3) // 4 * 4), dtype=torch.float32, device=x.device)
        ops.linear(x.reshape(rows, x.shape[-1]), weight, out=buf[:, :N])
        return buf[:, :N].view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy2 = dy if dy.dim() == 2 else dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != torch.bfloat16 or dy2.stride(1) != 1 or dy2.stride(0) % 8:
            padded = torch.zeros((dy2.shape[0], (dy2.shape[1] + 7) // 8 * 8), dtype=torch.bfloat16, device=dy2.device)
            padded[:, :dy2.shape[1]] = dy2
            dy2 = padded[:, :dy.shape[-1]]
        x2 = x.reshape(-1, x.shape[-1])
        dx = ops.gemm_tn(dy2, w, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        # wgrad: fp32 accumulation in registers, ONE rounding to the parameter dtype in the epilogue (== fp32 result .to(bf16))
        dw = None
        if ctx.needs_input_grad[1]:
            dw = ops.gemm_tn(dy2, x2, a_mn=True, b_mn=True, out_dtype=torch.bfloat16 if w.dtype == torch.bfloat16 else torch.float32)
            dw = dw if dw.dtype == w.dtype else dw.to(w.dtype)
        return dx, dw, None, (dy if ctx.has_res else None)


class RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        ctx.save_for_backward(x, weight)
        ctx.eps = eps
        return ops.rmsnorm(x, weight, eps)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx, dw = rmsnorm_bwd(x.reshape(-1, x.shape[-1]), w, dy.reshape(-1, dy.shape[-1]).contiguous(), ctx.eps)
        return dx.view(x.shape), dw.to(w.dtype), None


class RopeFn(torch.autograd.Function):
    """Rotate-half RoPE on the first `heads` heads of the packed [tokens, width] rows (q and k of the packed qkv).  Stand-alone
    (out-of-place) form; the decoder uses QKVRopeFn, which rotates in place inside the projection's autograd node."""

    @staticmethod
    def forward(ctx, qkv2, cos, sin, heads, head_dim, neg_sin=None):
        ctx.save_for_backward(cos, sin if neg_sin is None else neg_sin)
        ctx.heads, ctx.head_dim, ctx.have_neg = heads, head_dim, neg_sin is not None
        out = qkv2.clone()
        ops.rope_(out, cos, sin, heads, head_dim)
        return out

    @staticmethod
    def backward(ctx, dy):
        cos, s_ = ctx.saved_tensors
        nsin = s_ if ctx.have_neg else (-s_).contiguous()
        g = dy.clone()
        ops.rope_(g, cos, nsin, ctx.heads, ctx.head_dim)                          # R(theta)^T = R(-theta)
        return g, None, None, None, None, None


class QKVRopeFn(torch.autograd.Function):
    """Packed q|k|v projection + rotate-half RoPE on the q and k heads as one autograd node: the rotation runs in place on
    the fresh GEMM output (forward) and on the incoming packed gradient (backward: R(theta)^T = R(-theta), then the
    dgrad / wgrad GEMMs) -- no clone of the [tokens, 3H] tensor either way."""

    @staticmethod
    def forward(ctx, x2, weight, cos, sin, neg_sin, heads, head_dim):
        qkv = ops.linear(x2, weight)
        ops.rope_(qkv, cos, sin, heads, head_dim)
        ctx.save_for_backward(x2, weight, cos, neg_sin)
        ctx.heads, ctx.head_dim = heads, head_dim
        return qkv

    @staticmethod
    def backward(ctx, dy):
        x2, w, cos, neg_sin = ctx.saved_tensors
        g = dy if (dy.dim() == 2 and dy.stride(1) == 1 and dy.stride(0) % 8 == 0) else dy.reshape(dy.shape[0], -1).contiguous()
        ops.rope_(g, cos, neg_sin, ctx.heads, ctx.head_dim)                       # in place: this edge owns the gradient
        dx = ops.gemm_tn(g, w, b_mn=True) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            dw = ops.gemm_tn(g, x2, a_mn=True, b_mn=True, out_dtype=torch.bfloat16 if w.dtype == torch.bfloat16 else torch.float32)
            dw = dw if dw.dtype == w.dtype else dw.to(w.dtype)
        return dx, dw, None, None, None, None, None


class CausalAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale):
        ctx.save_for_backward(q, k, v)
        ctx.scale = scale
        return ops.attention(q, k, v, causal=True, scale=scale)

    @staticmethod
    def backward(ctx, dctx):
        q, k, v = ctx.saved_tensors
        B, T, H, D = q.shape
        dq, dk, dv = attention_backward(q, k, v, dctx.reshape(B, T, H, D), ctx.scale)
        return dq, dk, dv, None


class CausalAttentionPackedFn(torch.autograd.Function):
    """Causal attention on the packed projection output qkv5 [B, T, G + 2, nkv, D] (G query heads per KV head; MHA:
    [B, T, 3, H, D]): the forward reads q / k / v as strided views (no copies), the backward returns the packed gradient
    (attention_backward_packed)."""

    @staticmethod
    def forward(ctx, qkv5, scale):
        ctx.save_for_backward(qkv5)
        ctx.scale = scale
        G = qkv5.shape[2] - 2
        return ops.attention(qkv5[:, :, :G].flatten(2, 3), qkv5[:, :, G], qkv5[:, :, G + 1], causal=True, scale=scale)

    @staticmethod
    def backward(ctx, dctx):
        (qkv5,) = ctx.saved_tensors
        return attention_backward_packed(qkv5, dctx, ctx.scale), None


class SwiGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gu):
        ctx.save_for_backward(gu)
        return swiglu_fwd(gu)

    @staticmethod
    def backward(ctx, dh):
        (gu,) = ctx.saved_tensors
        return swiglu_bwd(gu, dh.contiguous())


class CrossEntropyFn(torch.autograd.Function):
    """mean CE of fp32 logits [rows, V] over the rows whose label is in [0, V) (-100 and any other label outside the
    vocabulary are ignored, the same rows as `ops.ce_loss` and the kernel); loss and dlogits from one kernel.  When every
    row is ignored the loss is 0 with a zero gradient (torch and `ops.ce_loss` give nan), so that a micro-batch without
    text positions adds nothing to an accumulated step."""

    @staticmethod
    def forward(ctx, logits, labels):
        rows, V = logits.shape
        n_valid = ((labels >= 0) & (labels < V)).sum().to(torch.int64).reshape(1)
        loss_sum = torch.zeros(1, dtype=torch.float32, device=logits.device)
        # bf16 rows with a 16-byte pitch, so the lm_head dgrad / wgrad GEMMs read dlogits in place (TMA operand)
        dlogits = torch.empty((rows, (V + 7) // 8 * 8), dtype=torch.bfloat16, device=logits.device)[:, :V]
        with torch.cuda.device(logits.device):
            rc = _lib.lib().vllm_ce_loss_f32(logits.data_ptr(), logits.stride(0), labels.data_ptr(), n_valid.data_ptr(), rows, V,
                                             loss_sum.data_ptr(), dlogits.data_ptr(), dlogits.stride(0), ops._stream())
        _lib.check(rc, "vllm_ce_loss_f32")
        ctx.save_for_backward(dlogits)
        return (loss_sum / n_valid.clamp(min=1).float()).reshape(())

    @staticmethod
    def backward(ctx, dloss):
        (dlogits,) = ctx.saved_tensors
        # in place, keeping the padded pitch: dlogits * dloss in fp32 with one rounding (dloss = 1 leaves every byte as it
        # is; a bf16 dloss would bias every gradient, e.g. by +0.2 % for bf16(1/3) under 3-way gradient accumulation)
        scale = dloss.detach().to(torch.float32).reshape(1).contiguous()
        rows, V = dlogits.shape
        with torch.cuda.device(dlogits.device):
            rc = _lib.lib().vllm_scale_rows_bf16(dlogits.data_ptr(), dlogits.stride(0), rows, V, scale.data_ptr(), ops._stream())
        _lib.check(rc, "vllm_scale_rows_bf16")
        return dlogits, None


# ---- the trainable decoders ---------------------------------------------------------------------------------------------
def decoder_layer_train(x, cos, sin, neg_sin, norm1_w, norm2_w, eps, wqkv, wo, w_gate_up, w_down, nq, nkv, D):
    """fwd of one pre-norm decoder layer as autograd Functions on this repo's kernels, on the layer's (packed) weights --
    shared by the Llama and InternLM2 training wrappers, as llama.decoder_layer_forward is by the inference modules:
    RMSNorm, q|k|v GEMM + RoPE on the nq + nkv q and k heads, causal (grouped-query) attention, O GEMM (+ residual in the
    epilogue), RMSNorm, gate|up GEMM, SwiGLU, down GEMM (+ residual)."""
    B, T, H = x.shape
    h = RMSNormFn.apply(x, norm1_w, eps)
    qkv = QKVRopeFn.apply(h.view(B * T, H), wqkv, cos, sin, neg_sin, nq + nkv, D).view(B, T, nq // nkv + 2, nkv, D)
    ctx = CausalAttentionPackedFn.apply(qkv, D ** -0.5)
    x = LinearFn.apply(ctx, wo, False, x)                                             # + residual in the GEMM epilogue
    h = RMSNormFn.apply(x, norm2_w, eps)
    gu = LinearFn.apply(h, w_gate_up)
    act = SwiGLUFn.apply(gu.view(B * T, -1)).view(B, T, -1)
    return LinearFn.apply(act, w_down, False, x)


class _DecoderTrain(nn.Module):
    """fwd+bwd of a decoder stack on the parameters of an inference module (shared, not copied); sequence length a multiple
    of 256.  A subclass names the weights: layer_weights(layer) -> (norm1, norm2, wqkv, wo, w_gate_up, w_down), where
    wqkv / w_gate_up are differentiable functions of the module's parameters (so the gradients land on them), and
    final_weights() -> (final norm, lm head)."""

    def __init__(self, lm, nq, nkv, D, eps, theta):
        super().__init__()
        self.lm = lm
        self.nq, self.nkv, self.D, self.eps, self.theta = nq, nkv, D, eps, theta
        if nq % nkv:
            raise NotImplementedError("num_attention_heads must be a multiple of num_key_value_heads")

    def forward(self, inputs_embeds, labels=None):
        B, T, H = inputs_embeds.shape
        pos = torch.arange(T, device=inputs_embeds.device)[None].expand(B, T)
        cos, sin = rope_tables(pos, self.D, self.theta, inputs_embeds.dtype)
        neg_sin = (-sin).contiguous()
        x = inputs_embeds
        for layer in self.layers():
            n1, n2, wqkv, wo, wgu, wdown = self.layer_weights(layer)
            x = decoder_layer_train(x, cos, sin, neg_sin, n1, n2, self.eps, wqkv, wo, wgu, wdown, self.nq, self.nkv, self.D)
        norm_w, head_w = self.final_weights()
        hidden = RMSNormFn.apply(x, norm_w, self.eps)
        # fp32 logits like `logits.float()` (mv2.py:738), as a 2-D [B*T, V] view of a pitch-padded buffer so that the loss
        # kernel and the lm_head backward GEMMs read logits / dlogits in place
        logits2 = LinearFn.apply(hidden.view(B * T, H), head_w, True)
        loss = None
        if labels is not None:                                                             # mv2.py:741-757: shift, flatten, CE
            # "shift so that tokens < n predict n": instead of slicing the 1.5 GB logits, shift the labels and ignore the
            # last position of every row -- the same set of (logit row, label) pairs, the same mean
            shift_labels = torch.cat([labels[:, 1:], torch.full_like(labels[:, :1], -100)], 1).reshape(-1).contiguous()
            loss = CrossEntropyFn.apply(logits2, shift_labels)
        return loss, logits2.view(B, T, -1), hidden


class B200LlamaForCausalLMTrain(_DecoderTrain):
    """fwd+bwd of the decoder stack on the parameters of a `B200LlamaForCausalLM` (HF names; MHA like Vicuna-7B or
    grouped-query attention)."""

    def __init__(self, lm):
        cfg = lm.config
        H, nq = cfg.hidden_size, cfg.num_attention_heads
        super().__init__(lm, nq, getattr(cfg, "num_key_value_heads", None) or nq, H // nq, cfg.rms_norm_eps,
                         getattr(cfg, "rope_theta", None) or 10000.0)
        self.H = H

    def _packed(self, layer):
        """[(nq + 2 nkv) D, H] packed q|k|v weight and [2I, H] row-interleaved gate|up weight as differentiable functions of
        the layer's parameters (torch.cat / stack are autograd-tracked, so the gradients land on q_proj ... up_proj)."""
        a, m = layer.self_attn, layer.mlp
        wqkv = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)
        wgu = torch.stack([m.gate_proj.weight, m.up_proj.weight], 1).reshape(2 * m.gate_proj.weight.shape[0], self.H)
        return wqkv, wgu

    def layers(self):
        return self.lm.model.layers

    def layer_weights(self, layer):
        wqkv, wgu = self._packed(layer)
        return (layer.input_layernorm.weight, layer.post_attention_layernorm.weight, wqkv, layer.self_attn.o_proj.weight,
                wgu, layer.mlp.down_proj.weight)

    def final_weights(self):
        return self.lm.model.norm.weight, self.lm.lm_head.weight


class B200InternLM2ForCausalLMTrain(_DecoderTrain):
    """fwd+bwd of the decoder stack on the parameters of a `B200InternLM2ForCausalLM` (the reference's names: the 26B
    preset's InternLM2-20B, 48 query heads over 8 KV heads).  The fused `attention.wqkv` interleaves (G query heads, k, v)
    per KV head along its rows; its rows are gathered into q | k | v by an autograd-tracked index, so the gradient lands
    on `wqkv` in the reference's interleaved order.  The loss is that of B200LlamaForCausalLMTrain."""

    def __init__(self, lm):
        cfg = lm.config
        if getattr(cfg, "rope_scaling", None) is not None:
            raise NotImplementedError("InternLM2 rope_scaling (linear / dynamic NTK) is not on the reference's path")
        if bool(getattr(cfg, "bias", False)):
            raise NotImplementedError("InternLM2 with bias=True: the training path has no bias gradients")
        H, nq = cfg.hidden_size, cfg.num_attention_heads
        nkv = getattr(cfg, "num_key_value_heads", None) or nq
        super().__init__(lm, nq, nkv, H // nq, cfg.rms_norm_eps, getattr(cfg, "rope_theta", None) or 10000.0)
        G, D = nq // nkv, H // nq
        idx = torch.arange((nq + 2 * nkv) * D).view(nkv, G + 2, D)                    # wqkv row of (kv head, slot, d)
        self._perm = torch.cat([idx[:, :G].reshape(-1), idx[:, G].reshape(-1), idx[:, G + 1].reshape(-1)])
        self._perm_dev = {}

    def layers(self):
        return self.lm.model.layers

    def layer_weights(self, layer):
        a, f = layer.attention, layer.feed_forward
        w = a.wqkv.weight
        perm = self._perm_dev.get(w.device)
        if perm is None:
            perm = self._perm_dev[w.device] = self._perm.to(w.device)
        wqkv = w[perm]                                                                # q | k | v rows; backward scatters back
        wgu = torch.stack([f.w1.weight, f.w3.weight], 1).reshape(2 * f.w1.weight.shape[0], f.w1.weight.shape[1])
        return layer.attention_norm.weight, layer.ffn_norm.weight, wqkv, a.wo.weight, wgu, f.w2.weight

    def final_weights(self):
        return self.lm.model.norm.weight, self.lm.output.weight
