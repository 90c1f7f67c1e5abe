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
from .llama import right_padding_lengths, rope_tables


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


def _partials(rows, cols, n, device):
    n_part = _lib.lib().vllm_rmsnorm_bwd_partials(rows)
    return n_part, torch.empty((n * max(n_part, 1), cols), dtype=torch.float32, device=device)


def gelu_fwd(u):
    y = torch.empty_like(u)
    with torch.cuda.device(u.device):
        rc = _lib.lib().vllm_gelu_fwd_bf16(u.data_ptr(), u.stride(0), y.data_ptr(), y.stride(0), u.shape[0], u.shape[1], ops._stream())
    _lib.check(rc, "vllm_gelu_fwd_bf16")
    return y


def gelu_bwd(u, dy):
    dx = torch.empty_like(u)
    with torch.cuda.device(u.device):
        rc = _lib.lib().vllm_gelu_bwd_bf16(u.data_ptr(), u.stride(0), dy.data_ptr(), dy.stride(0), dx.data_ptr(), dx.stride(0),
                                           u.shape[0], u.shape[1], ops._stream())
    _lib.check(rc, "vllm_gelu_bwd_bf16")
    return dx


def bias_grad(dy2):
    """fp32 column sums of dy [rows, N] (bf16, unit inner stride), in a fixed order (vllm_bias_grad_bf16)."""
    rows, cols = dy2.shape
    n_part, part = _partials(rows, cols, 1, dy2.device)
    db = torch.empty(cols, dtype=torch.float32, device=dy2.device)
    with torch.cuda.device(dy2.device):
        rc = _lib.lib().vllm_bias_grad_bf16(dy2.data_ptr(), dy2.stride(0), db.data_ptr(), part.data_ptr(), n_part, rows, cols,
                                            ops._stream())
    _lib.check(rc, "vllm_bias_grad_bf16")
    return db


def layernorm_bwd_wb(x2, dy2, eps):
    """nn.LayerNorm weight / bias gradients (fp32, fixed summation order; vllm_layernorm_bwd_wb_bf16) -- no dx."""
    rows, cols = x2.shape
    n_part, part = _partials(rows, cols, 2, x2.device)
    dw = torch.empty(cols, dtype=torch.float32, device=x2.device)
    db = torch.empty(cols, dtype=torch.float32, device=x2.device)
    with torch.cuda.device(x2.device):
        rc = _lib.lib().vllm_layernorm_bwd_wb_bf16(x2.data_ptr(), x2.stride(0), dy2.data_ptr(), dy2.stride(0), dw.data_ptr(),
                                                   db.data_ptr(), part.data_ptr(), n_part, rows, cols, float(eps), ops._stream())
    _lib.check(rc, "vllm_layernorm_bwd_wb_bf16")
    return dw, db


def layernorm_gelu_bwd(x2, weight, bias, dy2, eps):
    """Backward of ops.layernorm(..., gelu=True) on [rows, cols] bf16 rows: dx (bf16) and fp32 weight / bias gradients
    summed in a fixed order (vllm_layernorm_gelu_bwd_bf16)."""
    rows, cols = x2.shape
    L = _lib.lib()
    n_part = L.vllm_layernorm_gelu_bwd_partials(rows)
    part = torch.empty((2 * max(n_part, 1), cols), dtype=torch.float32, device=x2.device)
    dx = torch.empty_like(x2)
    dw = torch.empty(cols, dtype=torch.float32, device=x2.device)
    db = torch.empty(cols, dtype=torch.float32, device=x2.device)
    with torch.cuda.device(x2.device):
        rc = L.vllm_layernorm_gelu_bwd_bf16(x2.data_ptr(), x2.stride(0), weight.data_ptr(), bias.data_ptr(), dy2.data_ptr(),
                                            dy2.stride(0), dx.data_ptr(), dx.stride(0), dw.data_ptr(), db.data_ptr(),
                                            part.data_ptr(), n_part, rows, cols, float(eps), ops._stream())
    _lib.check(rc, "vllm_layernorm_gelu_bwd_bf16")
    return dx, dw, db


def point_pool_bwd(loc, wgt, grad, h, w):
    """Backward of the region encoder's point pooling over `levels` feature levels of one map: loc [levels, R, n, 2] /
    wgt [levels, R, n] fp32 point tables (region_encoder.point_table, padded to one n), grad [levels, R, C] bf16 ->
    d(map) [R, h * w, C] bf16 = sum_l a_l (x) grad_l / count_l (vllm_point_pool_bwd_bf16)."""
    levels, R, n = wgt.shape
    C = grad.shape[-1]
    cnt = wgt.sum(2).contiguous()                                   # the forward's counts (wgt.sum(1) per level)
    out = torch.empty((R, h * w, C), dtype=torch.bfloat16, device=grad.device)
    density = torch.empty((levels, R, h * w), dtype=torch.float32, device=grad.device)
    with torch.cuda.device(grad.device):
        rc = _lib.lib().vllm_point_pool_bwd_bf16(loc.data_ptr(), wgt.data_ptr(), cnt.data_ptr(), n, grad.data_ptr(), levels, R,
                                                 h, w, C, density.data_ptr(), out.data_ptr(), ops._stream())
    _lib.check(rc, "vllm_point_pool_bwd_bf16")
    return out


def assemble_embeds_bwd(plan, d_embeds, source_rows, wanted):
    """Gradients of ops.assemble_embeds' sources from d(inputs_embeds) [B, L, C]: `source_rows` = rows of (token table, det
    table, pose table, image features), `wanted` = which of them need a gradient.  Positions are sorted stably by destination
    row (torch.sort, glue) and one segment-sum kernel (vllm_assemble_embeds_bwd_bf16) writes every wanted source: fp32 sums
    in position order, rows no position names exact 0.  Returns one tensor (or None) per source."""
    C = d_embeds.shape[-1]
    base, offs = 0, []
    for n, w in zip(source_rows, wanted):
        offs.append(base if w else None)
        base += n if w else 0
    if base == 0:
        return [None] * 4
    big = torch.iinfo(torch.int32).max                             # positions of unwanted sources sort past every row
    lut = torch.tensor([o if o is not None else big for o in offs], dtype=torch.int64, device=d_embeds.device)
    dest = torch.minimum(lut[plan.kind.reshape(-1).long()] + plan.row.reshape(-1).long(), lut.new_tensor(big))
    dest, order = torch.sort(dest.to(torch.int32), stable=True)
    order = order.to(torch.int32)
    dy = d_embeds.reshape(-1, C)
    dy = dy if dy.is_contiguous() and dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16).contiguous()
    out = torch.empty((base, C), dtype=torch.bfloat16, device=d_embeds.device)
    with torch.cuda.device(out.device):
        rc = _lib.lib().vllm_assemble_embeds_bwd_bf16(dest.data_ptr(), order.data_ptr(), dest.numel(), dy.data_ptr(), C,
                                                      out.data_ptr(), base, ops._stream())
    _lib.check(rc, "vllm_assemble_embeds_bwd_bf16")
    return [out[o:o + n] if o is not None else None for o, n in zip(offs, source_rows)]


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


def head_stack_qkv_pad(rows, nq, nkv, D, T_pad, stacks=None):
    """head_stack_qkv with T_pad >= T rows per (batch, head) matrix (vllm_head_stack_qkv_pad_bf16): rows T .. T_pad - 1 of
    every stacked matrix are zeros; the inverse skips them.  nkv = 0 stacks the nq heads of a plain [B, T, nq D] tensor."""
    B, T = rows.shape[0], rows.shape[1]
    to_stacked = stacks is None
    if to_stacked:
        stacks = torch.empty(((nq + 2 * nkv) * B * T_pad, D), dtype=rows.dtype, device=rows.device)
    nq_rows, nkv_rows = B * nq * T_pad, B * nkv * T_pad
    q, k, v = stacks[:nq_rows], stacks[nq_rows:nq_rows + nkv_rows], stacks[nq_rows + nkv_rows:]
    with torch.cuda.device(rows.device):
        rc = _lib.lib().vllm_head_stack_qkv_pad_bf16(rows.data_ptr(), rows.stride(1), q.data_ptr(),
                                                     k.data_ptr() if nkv else None, v.data_ptr() if nkv else None, B, T, T_pad,
                                                     nq, nkv, D, 1 if to_stacked else 0, ops._stream())
    _lib.check(rc, "vllm_head_stack_qkv_pad_bf16")
    return stacks if to_stacked else rows


def attention_backward_packed(qkv5, do, scale, seqlens=None):
    """Backward of causal softmax(q k^T * scale) v for the PACKED projection output qkv5 [B, T, G + 2, nkv, D] (bf16: the
    nq = G * nkv query heads, then the nkv key heads, then the nkv value heads of a row; q head i attends with KV head
    i // G, as HF's repeat_kv; MHA is G = 1, [B, T, 3, H, D]) and do [B, T, nq*D].  Returns d(qkv5) in the same packed
    layout.  The (batch, head) matrices are stacked along rows for the block-diagonal batched GEMMs by ONE copy of qkv5
    (and one of do); the three gradient GEMMs write one stacked buffer that ONE copy turns back into the packed layout.
    Grouped-query attention needs no repeated K / V: S, dP and dQ read KV matrix i // G, and dK, dV reduce over the G
    query matrices of a KV head inside one GEMM (fp32 accumulation, one rounding).

    seqlens (int32 [B], right padding) or a T that is not a multiple of 256 takes the padded form: every matrix is stacked
    with T_pad = roundup(T, 256) rows (zeros past T), the softmax gives P = 0 for keys j >= seqlens[b] (HF's mask: key j is
    visible to query i iff j <= i and j < len, for every query row), and with P = 0 the softmax backward gives dS = 0 there,
    so the same five GEMMs and dS kernel serve."""
    B, T, parts, nkv, D = qkv5.shape
    G = parts - 2
    if G < 1 or D % 64:
        raise RuntimeError("attention_backward: head_dim must be a multiple of 64")
    padded = seqlens is not None or T % 256 != 0
    Tp = (T + 255) // 256 * 256
    nq = G * nkv
    BQ, BKV = B * nq, B * nkv
    rows = qkv5.reshape(B, T, -1)                                               # a view for the decoder's packed projection
    if rows.stride(2) != 1 or rows.stride(1) % 8 or rows.data_ptr() % 16:
        rows = rows.contiguous()
    if padded:
        stk = head_stack_qkv_pad(rows, nq, nkv, D, Tp)
        dos = head_stack_qkv_pad(do.reshape(B, T, nq * D).contiguous(), nq, 0, D, Tp)
    else:
        stk = head_stack_qkv(rows, nq, nkv, D)                                  # Q | K | V stacks, [(b, h), T, D] each
        dos = head_stack(do, B, T, 1, nq, D, True).view(BQ * T, D)
    qs, ks, vs = stk[:BQ * Tp], stk[BQ * Tp:(BQ + BKV) * Tp], stk[(BQ + BKV) * Tp:]
    L_ = _lib.lib()
    p = gemm_batched(qs, ks, BQ, Tp, Tp, D, causal=1, group=G)                   # S = Q K^T, tiles above the diagonal skipped
    with torch.cuda.device(qkv5.device):
        if padded:
            # lengths past T are T, as in the forward kernel (min(seqlens[b], Tk)): the zero rows T .. T_pad stay masked
            lens = (seqlens.clamp(max=T) if seqlens is not None else
                    torch.full((B,), T, dtype=torch.int32, device=qkv5.device))
            rc = L_.vllm_softmax_causal_len_bf16(p.data_ptr(), p.stride(0), BQ, nq, Tp, lens.data_ptr(), float(scale), ops._stream())
            _lib.check(rc, "vllm_softmax_causal_len_bf16")
        else:
            _lib.check(L_.vllm_softmax_causal_bf16(p.data_ptr(), p.stride(0), BQ, T, float(scale), ops._stream()),
                       "vllm_softmax_causal_bf16")
    dp = gemm_batched(dos, vs, BQ, Tp, Tp, D, causal=1, group=G)                 # dP = dO V^T
    with torch.cuda.device(qkv5.device):
        _lib.check(L_.vllm_attn_ds_bf16(p.data_ptr(), dp.data_ptr(), p.stride(0), BQ, Tp, float(scale), ops._stream()), "vllm_attn_ds_bf16")
    ds = dp
    dstk = torch.empty_like(stk)
    dqs, dks, dvs = dstk[:BQ * Tp], dstk[BQ * Tp:(BQ + BKV) * Tp], dstk[(BQ + BKV) * Tp:]
    gemm_batched(p, dos, BQ, Tp, D, Tp, a_mn=True, b_mn=True, causal=2, out=dvs, group=G, reduce=True)   # dV = sum_g P_g^T dO_g
    gemm_batched(ds, qs, BQ, Tp, D, Tp, a_mn=True, b_mn=True, causal=2, out=dks, group=G, reduce=True)   # dK = sum_g dS_g^T Q_g
    gemm_batched(ds, ks, BQ, Tp, D, Tp, b_mn=True, causal=3, out=dqs, group=G)                            # dQ = dS K
    dqkv = torch.empty((B, T, parts * nkv * D), dtype=qkv5.dtype, device=qkv5.device)
    if padded:
        return head_stack_qkv_pad(dqkv, nq, nkv, D, Tp, stacks=dstk).view(B, T, parts, nkv, D)
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
    def forward(ctx, x, weight, out_f32=False, residual=None, bias=None):
        ctx.save_for_backward(x, weight)
        ctx.has_res = residual is not None
        if not out_f32:
            return ops.linear(x, weight, bias=bias, residual=residual)   # y = x W^T (+ bias, + residual in the GEMM epilogue)
        assert residual is None and bias is None
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
        db = bias_grad(dy2).to(w.dtype) if len(ctx.needs_input_grad) > 4 and ctx.needs_input_grad[4] else None
        return dx, dw, None, (dy if ctx.has_res else None), db


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
    (attention_backward_packed).  seqlens: int32 [B] key lengths of a right-padded batch, or None."""

    @staticmethod
    def forward(ctx, qkv5, scale, seqlens=None):
        ctx.save_for_backward(qkv5)
        ctx.scale, ctx.seqlens = scale, seqlens
        G = qkv5.shape[2] - 2
        return ops.attention(qkv5[:, :, :G].flatten(2, 3), qkv5[:, :, G], qkv5[:, :, G + 1], causal=True, scale=scale,
                             seqlens=seqlens)

    @staticmethod
    def backward(ctx, dctx):
        (qkv5,) = ctx.saved_tensors
        if ctx.seqlens is None:
            return attention_backward_packed(qkv5, dctx, ctx.scale), None, None
        return attention_backward_packed(qkv5, dctx, ctx.scale, ctx.seqlens), None, None


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
def decoder_layer_train(x, cos, sin, neg_sin, norm1_w, norm2_w, eps, wqkv, wo, w_gate_up, w_down, nq, nkv, D, seqlens=None):
    """fwd of one pre-norm decoder layer as autograd Functions on this repo's kernels, on the layer's (packed) weights --
    shared by the Llama and InternLM2 training wrappers, as llama.decoder_layer_forward is by the inference modules:
    RMSNorm, q|k|v GEMM + RoPE on the nq + nkv q and k heads, causal (grouped-query) attention, O GEMM (+ residual in the
    epilogue), RMSNorm, gate|up GEMM, SwiGLU, down GEMM (+ residual).  seqlens: key lengths of a right-padded batch."""
    B, T, H = x.shape
    h = RMSNormFn.apply(x, norm1_w, eps)
    qkv = QKVRopeFn.apply(h.view(B * T, H), wqkv, cos, sin, neg_sin, nq + nkv, D).view(B, T, nq // nkv + 2, nkv, D)
    ctx = CausalAttentionPackedFn.apply(qkv, D ** -0.5, seqlens)
    x = LinearFn.apply(ctx, wo, False, x)                                             # + residual in the GEMM epilogue
    h = RMSNormFn.apply(x, norm2_w, eps)
    gu = LinearFn.apply(h, w_gate_up)
    act = SwiGLUFn.apply(gu.view(B * T, -1)).view(B, T, -1)
    return LinearFn.apply(act, w_down, False, x)


class _DecoderTrain(nn.Module):
    """fwd+bwd of a decoder stack on the parameters of an inference module (shared, not copied); any sequence length, and
    right-padded batches through `attention_mask` (HF semantics: key j is visible to query i iff j <= i and j < len[b],
    positions stay arange(T)).  A subclass names the weights: layer_weights(layer) -> (norm1, norm2, wqkv, wo, w_gate_up, w_down), where
    wqkv / w_gate_up are differentiable functions of the module's parameters (so the gradients land on them), and
    final_weights() -> (final norm, lm head)."""

    def __init__(self, lm, nq, nkv, D, eps, theta):
        super().__init__()
        self.lm = lm
        self.nq, self.nkv, self.D, self.eps, self.theta = nq, nkv, D, eps, theta
        if nq % nkv:
            raise NotImplementedError("num_attention_heads must be a multiple of num_key_value_heads")

    def forward(self, inputs_embeds, labels=None, attention_mask=None):
        B, T, H = inputs_embeds.shape
        seqlens = right_padding_lengths(attention_mask)                  # None when nothing is padded: the unmasked path
        pos = torch.arange(T, device=inputs_embeds.device)[None].expand(B, T)
        cos, sin = rope_tables(pos, self.D, self.theta, inputs_embeds.dtype)
        neg_sin = (-sin).contiguous()
        x = inputs_embeds
        for layer in self.layers():
            n1, n2, wqkv, wo, wgu, wdown = self.layer_weights(layer)
            x = decoder_layer_train(x, cos, sin, neg_sin, n1, n2, self.eps, wqkv, wo, wgu, wdown, self.nq, self.nkv, self.D,
                                    seqlens)
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


# ---- the multimodal chat step: vision-language bridge and sequence assembly with gradients -----------------------------
class GeluFn(torch.autograd.Function):
    """Exact-erf GELU (nn.GELU()) on the saved pre-activation u: y = gelu(u), du = dy * gelu'(u)."""

    @staticmethod
    def forward(ctx, u):
        ctx.save_for_backward(u)
        return gelu_fwd(u)

    @staticmethod
    def backward(ctx, dy):
        (u,) = ctx.saved_tensors
        return gelu_bwd(u, dy.contiguous())


class LayerNormWBFn(torch.autograd.Function):
    """nn.LayerNorm whose input takes no gradient (the frozen ViT's features): backward gives the weight / bias gradients."""

    @staticmethod
    def forward(ctx, x2, weight, bias, eps):
        if ctx.needs_input_grad[0]:
            raise NotImplementedError("LayerNorm backward to its input: the vision encoder must be frozen")
        ctx.save_for_backward(x2)
        ctx.eps = eps
        return ops.layernorm(x2, weight, bias, eps)

    @staticmethod
    def backward(ctx, dy):
        (x2,) = ctx.saved_tensors
        if not (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            return None, None, None, None
        dw, db = layernorm_bwd_wb(x2, dy.contiguous(), ctx.eps)
        return None, dw.to(torch.bfloat16), db.to(torch.bfloat16), None


class LayerNormGeluFn(torch.autograd.Function):
    """LayerNorm over the last dim followed by exact-erf GELU (the region encoder's LayerNorm2d -> GELU on channels-last
    rows), forward in one pass (ops.layernorm(gelu=True)), backward to the input, weight and bias in one pass."""

    @staticmethod
    def forward(ctx, x2, weight, bias, eps):
        ctx.save_for_backward(x2, weight, bias)
        ctx.eps = eps
        return ops.layernorm(x2, weight, bias, eps, gelu=True)

    @staticmethod
    def backward(ctx, dy):
        x2, w, b = ctx.saved_tensors
        dx, dw, db = layernorm_gelu_bwd(x2, w, b, dy.contiguous(), ctx.eps)
        return dx, dw.to(w.dtype), db.to(b.dtype), None


class RegionPoolFn(torch.autograd.Function):
    """The region encoder's levels: masks_out accumulates each level's frozen features on the embedding (bf16 adds, in
    level order) and every level pools it at its own points, exactly as B200RegionEncoder.forward.  Only the embedding takes
    a gradient: d(emb) = sum over levels of the pooling's transpose (point_pool_bwd), one kernel pass for all levels.
    emb [R, h, w, E]; feats: per level [R, h, w, E]; tables: per level (loc, wgt) of point_table.  -> [levels, R, E]."""

    @staticmethod
    def forward(ctx, emb, enc, feats, tables):
        masks_out, pooled = emb, []
        for f, (loc, wgt) in zip(feats, tables):
            masks_out = masks_out + f.to(masks_out.dtype)
            pooled.append(enc._pool_points(masks_out, loc, wgt))
        n = max(t[1].shape[1] for t in tables)
        loc = torch.stack([torch.nn.functional.pad(t[0], (0, 0, 0, n - t[0].shape[1])) for t in tables]).contiguous()
        wgt = torch.stack([torch.nn.functional.pad(t[1], (0, n - t[1].shape[1])) for t in tables]).contiguous()
        ctx.save_for_backward(loc, wgt)
        ctx.hw = emb.shape[1:3]
        return torch.stack(pooled)

    @staticmethod
    def backward(ctx, dpooled):
        loc, wgt = ctx.saved_tensors
        h, w = ctx.hw
        d = point_pool_bwd(loc, wgt, dpooled.to(torch.bfloat16).contiguous(), h, w)
        return d.view(d.shape[0], h, w, -1), None, None, None


def _conv_weight(conv, k_pad):
    """A Conv2d weight as the [Cout, Cin k k] GEMM operand (K zero-padded to k_pad), differentiable: its gradient lands on
    the native [Cout, Cin, k, k] parameter."""
    w = conv.weight.reshape(conv.out_channels, -1)
    return torch.nn.functional.pad(w, (0, k_pad - w.shape[1])) if k_pad != w.shape[1] else w


def region_encoder_train(enc, images, masks, image_features, sample_points=None):
    """fwd of a 'grid_sample' B200RegionEncoder as autograd Functions on this repo's kernels, with gradients for every
    parameter (mask_embedding.{0,1,3,4,6}, up_dim): the three convolutions are GEMMs over non-overlapping patches with the
    bias in the epilogue (LinearFn), LayerNorm2d -> GELU is one row pass each way (LayerNormGeluFn), the k2s2 patch
    rearrangement is a permute, the point pooling of every level is RegionPoolFn, up_dim one LinearFn per level, then the
    mean over levels.  The forward values are B200RegionEncoder.forward's bytes for the same points.  sample_points:
    [level][region] -> [n, 3] as the inference forward takes them; None draws them with rand_sample."""
    from .region_encoder import _patch_rows, point_table
    if enc.mask_pool_type != "grid_sample":
        raise NotImplementedError(f"region-encoder training with mask_pool_type={enc.mask_pool_type!r}: only 'grid_sample' "
                                  "(the reference's build_region_encoder builds no other)")
    me = enc.mask_embedding
    masks = masks.to(images.dtype)
    x = torch.cat([images, masks], dim=1).permute(0, 2, 3, 1)                               # [B, H, W, 4]
    B = x.shape[0]
    rows, h, w = _patch_rows(x, me[0].kernel_size[0])
    kp = (rows.shape[1] + 7) // 8 * 8
    rows = torch.nn.functional.pad(rows, (0, kp - rows.shape[1])) if kp != rows.shape[1] else rows
    y = LinearFn.apply(rows.contiguous(), _conv_weight(me[0], kp), False, None, me[0].bias)
    y = LayerNormGeluFn.apply(y, me[1].weight, me[1].bias, me[1].eps)
    rows, h, w = _patch_rows(y.view(B, h, w, -1), 2)
    y = LinearFn.apply(rows.contiguous(), _conv_weight(me[3], rows.shape[1]), False, None, me[3].bias)
    y = LayerNormGeluFn.apply(y, me[4].weight, me[4].bias, me[4].eps)
    y = LinearFn.apply(y, _conv_weight(me[6], y.shape[1]), False, None, me[6].bias)
    emb = y.view(B, h, w, -1)
    feats = []
    for f in image_features:
        f = f.reshape(B, h, w, -1) if f.dim() == 3 else f.permute(0, 2, 3, 1)
        assert f.shape[1:3] == (h, w)
        feats.append(f)
    pts = sample_points if sample_points is not None else enc.draw_points(masks, len(feats))
    tables = [point_table(p, emb.device) for p in pts[:len(feats)]]
    pooled = RegionPoolFn.apply(emb, enc, feats, tables)                                   # [levels, R, E]
    outs = [LinearFn.apply(pooled[l], enc.up_dim.weight, False, None, enc.up_dim.bias) for l in range(len(feats))]
    return torch.stack(outs).mean(dim=0)


class RegionScatterFn(torch.autograd.Function):
    """scatter_region_tokens with gradients: the forward writes the region features into the <region> rows; the backward
    gathers d(embeds) at those rows for the features (vllm_gather_rows_bf16) and zeroes them for the assembly -- the
    reference's inputs_embeds * (1 - region_mask) + features * region_mask, so no token-table row takes a gradient from a
    <region> position."""

    @staticmethod
    def forward(ctx, embeds, feats, input_ids, reg_token_id):
        from .modeling import scatter_region_tokens
        rows = torch.nonzero((input_ids == reg_token_id).reshape(-1)).reshape(-1)
        ctx.save_for_backward(rows)
        return scatter_region_tokens(input_ids, embeds, feats, reg_token_id)

    @staticmethod
    def backward(ctx, dy):
        (rows,) = ctx.saved_tensors
        B, L, C = dy.shape
        d = dy.clone(memory_format=torch.contiguous_format).view(B * L, C)         # one copy: dy itself stays as it is
        dfeat = ops.gather_rows(d, rows) if ctx.needs_input_grad[1] else None
        d[rows] = 0
        return d.view(B, L, C), dfeat, None, None


class AssembleEmbedsFn(torch.autograd.Function):
    """ops.assemble_embeds with gradients for the token table, the two [EMB] tables and the image features."""

    @staticmethod
    def forward(ctx, plan, embed_w, det_w, pose_w, feats, padding_idx=None):
        ctx.plan, ctx.padding_idx = plan, padding_idx
        ctx.rows = (embed_w.shape[0], det_w.shape[0], pose_w.shape[0], feats.shape[0] if feats is not None else 0)
        return ops.assemble_embeds(plan, embed_w, det_w, pose_w, feats)

    @staticmethod
    def backward(ctx, dy):
        want = list(ctx.needs_input_grad[1:5])
        grads = assemble_embeds_bwd(ctx.plan, dy, ctx.rows, want)
        if grads[0] is not None and ctx.padding_idx is not None:
            grads[0][ctx.padding_idx].zero_()                        # nn.Embedding(padding_idx=...): that row takes no gradient
        return (None, *grads, None)


def bridge_train(bridge, x2):
    """The vl_bridge (modeling.build_vl_bridge: `linear`, `mlpNx_gelu`, `internvl_mlp`) as autograd Functions on x2 [rows, in]:
    Linear = GEMM with the bias in the epilogue (dgrad / wgrad GEMMs, bias gradient kernel); a GELU after a Linear stores the
    pre-activation and applies GELU in its own pass; the LayerNorm of internvl_mlp runs unfused (weight / bias gradients)."""
    from .modeling import BridgeLayerNorm, BridgeLinear
    mods = [bridge] if isinstance(bridge, BridgeLinear) else list(bridge)
    x = x2
    for m in mods:
        if isinstance(m, BridgeLinear):
            x = LinearFn.apply(x, m.weight, False, None, m.bias)
        elif isinstance(m, nn.GELU):
            if m.approximate != "none":
                raise NotImplementedError("vl_bridge GELU: only the exact-erf form")
            x = GeluFn.apply(x)
        elif isinstance(m, BridgeLayerNorm):
            x = LayerNormWBFn.apply(x, m.weight, m.bias, m.eps)
        else:
            raise NotImplementedError(f"vl_bridge module {type(m).__name__} has no training path")
    return x


def _require_cuda_bf16(*tensors):
    """The step runs on CUDA tensors, floating-point ones in bfloat16."""
    for t in tensors:
        if t is not None and (not t.is_cuda or (t.is_floating_point() and t.dtype != torch.bfloat16)):
            raise NotImplementedError("the training step runs on CUDA tensors, floating-point ones in bfloat16")


def _bridge_input(model, hs):
    """[tiles, 1 + tokens, C] ViT hidden state -> the bridge's input rows (CLS dropped, pixel shuffle when configured)."""
    if model.use_pixelshuffle:
        x = ops.pixel_shuffle_rows(hs, 1)
    else:
        x = hs[:, 1:].contiguous()
    return x.reshape(-1, x.shape[-1])


class B200VisionLLMv2ModelTrain(nn.Module):
    """fwd+bwd of the reference's chat training step (train.py: `model(**batch)` then `loss.backward()`) on the parameters of
    a `B200VisionLLMv2Model` (shared, not copied): the frozen vision encoder under no_grad, the vl_bridge, the sequence
    assembly (token table, [EMB] tables, image features) and the LLM decoder with gradients, on right-padded batches.
    Modules frozen with the composite's freeze_* methods get no gradient and cost no weight-gradient GEMM.
    With `regions`, the region encoder runs on the frozen ViT's last three hidden states (region_encoder_train, or its
    inference forward after freeze_region_encoder()) and its features overwrite the <region> rows (RegionScatterFn);
    `region_sample_points` ([level][region] -> [n, 3]) replaces the random point draw, as in the inference forward.
    Refused (NotImplementedError): a trainable vision encoder, atom-tool losses (`targets`, `images_aug`), `regions` without
    a region encoder or with a pooling other than 'grid_sample', the [EMB] insert form, KV caches, caller-provided
    `inputs_embeds`, non-CUDA / non-bf16 batches."""

    def __init__(self, model):
        super().__init__()
        from .internlm2 import B200InternLM2ForCausalLM
        self.model = model
        lm = model.llm
        self.llm_train = B200InternLM2ForCausalLMTrain(lm) if isinstance(lm, B200InternLM2ForCausalLM) else B200LlamaForCausalLMTrain(lm)

    def forward(self, input_ids=None, inputs_embeds=None, attention_mask=None, images=None, images_aug=None, img_metas=None,
                targets=None, labels=None, past_key_values=None, use_cache=False, output_attentions=False,
                output_hidden_states=False, return_dict=True, regions=None, num_splits=None, region_sample_points=None,
                **unused):
        from .modeling import IGNORE_INDEX, VisionLLMv2ModelOutput
        m = self.model
        if past_key_values is not None or use_cache:
            raise NotImplementedError("training with a KV cache")
        if targets is not None or images_aug is not None:
            raise NotImplementedError("atom-tool losses (detection / pose / generation targets) have no training path")
        if regions is not None:
            if not getattr(m, "use_region_encoder", False):
                raise NotImplementedError("regions on a composite built without a region encoder")
            if m.region_encoder.mask_pool_type != "grid_sample":
                raise NotImplementedError("region-encoder training pools with 'grid_sample' only (the reference's "
                                          "build_region_encoder)")
        if inputs_embeds is not None or input_ids is None:
            raise NotImplementedError("the training step takes input_ids (the reference's collator batch)")
        _require_cuda_bf16(input_ids, m.llm.get_input_embeddings().weight,
                           *(images if isinstance(images, (list, tuple)) else [images]))
        feats, split_sizes = None, False
        if images is not None:
            if any(p.requires_grad for p in m.vis_encoder.parameters()):
                raise NotImplementedError("a trainable vision encoder: call freeze_vis_encoder() (the reference's default)")
            with torch.no_grad():
                hs, split_sizes, vit_out = m.vision_hidden_state(images)
            feats = bridge_train(m.vl_bridge, _bridge_input(m, hs))
        tokens_per_tile = 0
        if feats is not None:
            tiles = sum(split_sizes) if split_sizes is not None else hs.shape[0]
            tokens_per_tile = feats.shape[0] // tiles
        plan = ops.seq_index(input_ids, (m.det_tool_id, m.seg_tool_id, m.grd_tool_id), (m.pose_tool_id,), m.emb_token_id,
                             m.num_embs, m.imp_token_id, split_sizes if images is not None else False, tokens_per_tile)
        status = int(plan.status.item())
        if status & 1:
            raise NotImplementedError("the [EMB] insert form (tool tokens without pre-placed [EMB] slots) has no training path")
        if status & 2:
            raise RuntimeError("image token count mismatch between the <im_patch> slots and the ViT tokens")
        table = m.llm.get_input_embeddings()
        # the reference's token table is nn.Embedding(..., padding_idx=pad_token_id) (HF Llama, InternLM2)
        pad = table.padding_idx if table.padding_idx is not None else getattr(m.llm.config, "pad_token_id", None)
        embeds = AssembleEmbedsFn.apply(plan, table.weight, m.emb_embeddings_det.weight, m.emb_embeddings_pose.weight, feats,
                                        pad if pad is not None and 0 <= pad < table.weight.shape[0] else None)
        if regions is not None and images is not None:                                       # mv2.py:607-698
            from .modeling import region_encoder_inputs
            ri, rm, rf = region_encoder_inputs(images, regions, vit_out.hidden_states, split_sizes, num_splits)
            enc = m.region_encoder
            if any(p.requires_grad for p in enc.parameters()):
                rfeat = region_encoder_train(enc, ri, rm, rf, region_sample_points)
            else:                                                   # freeze_region_encoder(): the inference forward
                rfeat = enc(ri, rm, rf, sample_points=region_sample_points)
            embeds = RegionScatterFn.apply(embeds, rfeat, plan.new_ids, m.reg_token_id)
        if labels is not None:                                                               # mv2.py:740-757
            labels[(labels >= m.emb_token_id) & (labels <= m.emb_token_id + m.num_embs - 1)] = IGNORE_INDEX
        loss, logits, hidden = self.llm_train(embeds, labels=labels, attention_mask=attention_mask)
        return VisionLLMv2ModelOutput(loss=loss, logits=logits, last_hidden_state=hidden, input_ids=plan.new_ids)
