"""BASELINE cfg 5 as written: "LLM tensor-parallel=8 over NVLink ... fwd+bwd step" with "tensor-parallel QKV/O with a
single NCCL allreduce over NVLink per layer" (north_star) -- the training-side counterpart of tp.py.

Megatron split of the decoder layer over the ranks of a torch.distributed group:
  column-parallel  packed q|k|v rows of the rank's heads, gate|up rows of the rank's slice of the MLP width
  row-parallel     o_proj / down_proj columns of the same slices; their partial products are summed with ONE
                   `all_reduce` each (NCCL over NVLink / NVSwitch) -- two per layer in the forward
  replicated       the residual stream, both RMSNorms, the final norm and the lm_head (every rank holds all token rows)
The backward mirrors it through two tiny autograd Functions: `CopyToTP` (identity forward, all-reduce of the input
gradient backward) in front of the column-parallel GEMMs and `ReduceFromTP` (all-reduce forward, identity backward)
behind the row-parallel ones.  Every compute op in between is a kernel of this repo (train.py's Functions: wgmma GEMMs
with MN-major dgrad / wgrad, batched attention backward, RMSNorm / SwiGLU / RoPE / CE kernels); the collectives are NCCL
calls -- the peer-memory fusion of tp.py's forward exchange is not extended to the backward (DESIGN 10).

The op set is injected (`fns`) so that the host logic -- sharding, which gradients are all-reduced, loss replication --
runs on CPU over gloo with torch-native differentiable ops (tests/test_tp_train_cpu.py).
"""
import torch
import torch.distributed as dist
import torch.nn as nn


class CopyToTP(torch.autograd.Function):
    """Megatron's `f`: identity in the forward, all-reduce of the gradient in the backward."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dist.all_reduce(g, group=ctx.group)
        return g, None


class ReduceFromTP(torch.autograd.Function):
    """Megatron's `g`: all-reduce in the forward, identity in the backward."""

    @staticmethod
    def forward(ctx, x, group):
        x = x.contiguous()
        dist.all_reduce(x, group=group)
        return x

    @staticmethod
    def backward(ctx, g):
        return g, None


def kernel_fns():
    """The product op set: train.py's autograd Functions (this repo's kernels, forward and backward)."""
    from . import train as T
    return {"linear": lambda x, w: T.LinearFn.apply(x, w), "linear_f32": lambda x, w: T.LinearFn.apply(x, w, True),
            "rmsnorm": lambda x, w, eps: T.RMSNormFn.apply(x, w, eps),
            "rope": lambda qkv2, cos, sin, heads, D, neg_sin=None: T.RopeFn.apply(qkv2, cos, sin, heads, D, neg_sin),
            # projection + rotation as one node (in-place rotation of the fresh GEMM output / of the incoming gradient)
            "qkv_rope": lambda x2, w, cos, sin, neg_sin, heads, D: T.QKVRopeFn.apply(x2, w, cos, sin, neg_sin, heads, D),
            "attention": lambda q, k, v, scale: T.CausalAttentionFn.apply(q, k, v, scale),
            # packed [B, T, 3, H, D] projection output in, packed gradient out: no per-tensor copies (train.py)
            "attention_packed": lambda qkv5, scale: T.CausalAttentionPackedFn.apply(qkv5, scale),
            "swiglu": lambda gu2: T.SwiGLUFn.apply(gu2), "ce": lambda logits2, labels: T.CrossEntropyFn.apply(logits2, labels)}


def shard_for_training(sd, config, rank, world):
    """HF-named full state dict -> this rank's TRAINABLE shards (nn.Parameters): heads [r*nq/W, (r+1)*nq/W) of q|k|v and
    o_proj, MLP columns [r*I/W, (r+1)*I/W) of gate|up (row-interleaved like llama.LlamaMLP) and down_proj; norms,
    lm_head replicated."""
    nq = config.num_attention_heads
    nkv = getattr(config, "num_key_value_heads", None) or nq
    if nkv != nq:
        raise NotImplementedError("grouped-query attention backward")
    H = config.hidden_size
    D = H // nq
    inter = config.intermediate_size
    if nq % world or inter % world:
        raise ValueError(f"heads ({nq}) and MLP width ({inter}) must divide over {world} ranks")
    ql, il = nq // world * D, inter // world
    layers = []
    for i in range(config.num_hidden_layers):
        p = f"model.layers.{i}."
        g = sd[p + "mlp.gate_proj.weight"][rank * il:(rank + 1) * il]
        u = sd[p + "mlp.up_proj.weight"][rank * il:(rank + 1) * il]
        layers.append(nn.ParameterDict({
            "wqkv": nn.Parameter(torch.cat([sd[p + f"self_attn.{n}_proj.weight"][rank * ql:(rank + 1) * ql]
                                            for n in ("q", "k", "v")], 0).contiguous()),
            "wo": nn.Parameter(sd[p + "self_attn.o_proj.weight"][:, rank * ql:(rank + 1) * ql].contiguous()),
            "wgu": nn.Parameter(torch.stack([g, u], 1).reshape(2 * il, H).contiguous()),
            "wdown": nn.Parameter(sd[p + "mlp.down_proj.weight"][:, rank * il:(rank + 1) * il].contiguous()),
            "ln1": nn.Parameter(sd[p + "input_layernorm.weight"].clone()),
            "ln2": nn.Parameter(sd[p + "post_attention_layernorm.weight"].clone()),
        }))
    return nn.ModuleDict({"layers": nn.ModuleList(layers),
                          "top": nn.ParameterDict({"final_norm": nn.Parameter(sd["model.norm.weight"].clone()),
                                                   "lm_head": nn.Parameter(sd["lm_head.weight"].clone())})})


class TPLlamaTrain(nn.Module):
    """One rank of the tensor-parallel decoder, forward + backward.  forward(inputs_embeds [B, T, H], labels [B, T]) ->
    (loss, logits fp32 [B, T, V], hidden); every rank sees all tokens and computes the same loss.  After .backward():
    sharded weights hold their shard's gradient, replicated ones (norms, lm_head) the full gradient on every rank, and
    `inputs_embeds.grad` the full gradient."""

    def __init__(self, config, shards, group=None, fns=None, rope_tables=None):
        super().__init__()
        self.config, self.shards, self.group = config, shards, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.nq_local = config.num_attention_heads // self.world
        self.D = config.hidden_size // config.num_attention_heads
        self.eps = config.rms_norm_eps
        self.theta = getattr(config, "rope_theta", None) or 10000.0
        self.fns = fns or kernel_fns()
        if rope_tables is None:
            from .llama import rope_tables
        self.rope_tables = rope_tables

    def forward(self, inputs_embeds, labels=None):
        f, grp, W = self.fns, self.group, self.world
        B, T, H = inputs_embeds.shape
        nql, D = self.nq_local, self.D
        pos = torch.arange(T, device=inputs_embeds.device)[None].expand(B, T)
        cos, sin = self.rope_tables(pos, D, self.theta, inputs_embeds.dtype)
        packed = "attention_packed" in f                     # the kernel op set; torch-native test sets take q, k, v
        neg_sin = (-sin).contiguous() if packed else None
        tp_in = (lambda t: CopyToTP.apply(t, grp)) if W > 1 else (lambda t: t)
        tp_out = (lambda t: ReduceFromTP.apply(t, grp)) if W > 1 else (lambda t: t)
        x = inputs_embeds
        for ly in self.shards["layers"]:
            h = tp_in(f["rmsnorm"](x, ly["ln1"], self.eps))
            if packed:
                qkv = f["qkv_rope"](h.reshape(B * T, H), ly["wqkv"], cos, sin, neg_sin, 2 * nql, D).view(B, T, 3, nql, D)
                ctx = f["attention_packed"](qkv, D ** -0.5)
            else:
                qkv = f["linear"](h, ly["wqkv"])                                         # [B, T, 3 * nql * D]
                qkv = f["rope"](qkv.reshape(B * T, 3 * nql * D), cos, sin, 2 * nql, D).view(B, T, 3, nql, D)
                ctx = f["attention"](qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], D ** -0.5)
            x = x + tp_out(f["linear"](ctx.reshape(B, T, nql * D), ly["wo"]))            # ONE all-reduce (attention block)
            h = tp_in(f["rmsnorm"](x, ly["ln2"], self.eps))
            gu = f["linear"](h, ly["wgu"])
            act = f["swiglu"](gu.reshape(B * T, -1)).view(B, T, -1)
            x = x + tp_out(f["linear"](act, ly["wdown"]))                                # ONE all-reduce (MLP block)
        hidden = f["rmsnorm"](x, self.shards["top"]["final_norm"], self.eps)
        logits2 = f["linear_f32"](hidden.reshape(B * T, H), self.shards["top"]["lm_head"])
        loss = None
        if labels is not None:                                                           # mv2.py:741-757
            shift = torch.cat([labels[:, 1:], torch.full_like(labels[:, :1], -100)], 1).reshape(-1).contiguous()
            loss = f["ce"](logits2, shift)
        return loss, logits2.view(B, T, -1), hidden
