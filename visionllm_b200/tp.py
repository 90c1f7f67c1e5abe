"""Tensor-parallel Llama decoder over NVLink peer memory (BASELINE cfg 5, SURVEY.md 8e).

The reference runs HF ``LlamaForCausalLM`` unsharded inside ``VisionLLMv2Model.forward``
(visionllmv2/model/modeling_visionllmv2.py:724-738).  The north-star splits the LLM over the 8 GPUs of one NVSwitch
box "with a single all-reduce per layer".  This module is that split for `B200LlamaForCausalLM` (same config, same
HF state-dict names on the way in, same `inputs_embeds -> fp32 logits + last hidden state` contract):

* attention is tensor-parallel: rank r owns heads [r*nq/W, (r+1)*nq/W) -- column-parallel packed QKV, row-parallel
  o_proj;
* the residual stream, both RMSNorms and the MLP are sequence-parallel: rank r owns token rows [r*R, (r+1)*R) of the
  flattened [B*T, H] activation (R = B*T/W) and runs the whole gate|up / down projection on them (replicated MLP
  weights; the FLOPs per rank equal a column/row-parallel MLP, the second all-reduce of a Megatron layer disappears);
* the only exchange of a layer is therefore ONE reduce-scatter (o_proj partials -> row owners) + ONE all-gather
  (normalised rows -> everybody) = the volume of a single all-reduce, and neither is an NCCL call: the o_proj GEMM
  epilogue pushes its tiles into the owners' receive slots (`vllm_gemm_bf16_scatter`), and the fused
  reduce + residual + RMSNorm kernel pushes the normalised rows into every peer's gather buffer
  (`vllm_tp_reduce_norm_bf16`); arrival counters in peer memory order the kernels (csrc/peer.cu).

`PeerComm` owns the exchange buffer of one rank (cudaMalloc + CUDA IPC through the C-ABI; torch.distributed only
carries the 64-byte handles at setup).  `PeerComm.virtual(W, ...)` builds W ranks on ONE device whose pointer tables
cross-reference each other, and `run_lockstep` advances their forwards phase by phase on one stream -- the multi-rank
protocol (pointer tables, slots, counters, epochs) is then testable on a single GPU.

Why single buffers and ever-growing counters are safe (no per-layer barrier):
  * gather buffer: rank j writes its rows of epoch e+1 into rank i's gather buffer only after its reduce(e) kernel
    finished (stream order), which needed rank i's o_proj partials of epoch e, which rank i's stream issued after its
    QKV GEMM -- the last reader of the epoch-e gather buffer -- completed.  So nobody overwrites rows a peer still reads.
  * receive slots: rank i's o_proj of epoch e+1 runs after its wait for gather(e+1), i.e. after rank j's norm_push(e+1),
    which rank j's stream issued after its reduce(e) -- the last reader of its epoch-e slots -- completed.
  * counters: an arrival of epoch e+1 can only be produced by a rank that has consumed every peer's epoch-e arrivals
    (same two chains), so "count >= e * arrivals_per_epoch" can never be satisfied by a mix of a fast rank's e+1 and a
    slow rank's missing e arrivals.  Comparisons are wrap-safe (signed difference).
  * across forwards the chain is broken (the final gather is read by host-ordered torch ops), hence the counter barrier
    at the top of `phases`.
A waiter that never sees its arrivals traps after 20 s (csrc/peer.cu) instead of hanging the GPU.

Forward only.  No CPU path: the collectives ARE the CUDA kernels; tests that run on CPU substitute a gloo-backed
double for the comm object (tests/test_tp_cpu.py).
"""
import ctypes
import os
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib, ops
from .llama import right_padding_lengths, rope_tables

_FLAG_BYTES = 4096
_GATHER_FLAG, _RECV_FLAG, _BARRIER_FLAG = 0, 256, 512      # byte offsets of the three arrival counters


class _DeviceBytes:
    """`__cuda_array_interface__` view of a raw device allocation so torch can wrap it without owning it."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False),
                                         "version": 2}


def _ptr_array(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(int(p)) for p in ptrs])


def exchange_bytes(rows_total, hidden, world):
    """Size of one rank's exchange buffer: counters | gather [M, H] bf16 | receive slots [W, M/W, H] bf16."""
    return _FLAG_BYTES + 2 * rows_total * hidden * 2


class PeerComm:
    """The exchange endpoint of one rank: its own buffer plus mapped pointers to every peer's buffer."""

    def __init__(self, rank, world, rows_total, hidden, device, own_ptr, peer_ptrs, owner=None):
        if rows_total % world:
            raise ValueError(f"token rows ({rows_total}) must divide over {world} ranks")
        self.rank, self.world, self.M, self.H = rank, world, rows_total, hidden
        self.R = rows_total // world
        if self.R % 128:
            raise ValueError("rows per rank must be a multiple of 128 (GEMM row tile)")
        if hidden % 64:
            raise ValueError("hidden size must be a multiple of 64")
        self.device = torch.device(device)
        self.base = [int(p) for p in peer_ptrs]            # base[j] = rank j's buffer as mapped in this process
        assert self.base[rank] == int(own_ptr)
        self._owner = owner                                 # keeps the allocation(s) alive
        nbytes = exchange_bytes(rows_total, hidden, world)
        raw = torch.as_tensor(_DeviceBytes(own_ptr, nbytes), device=self.device)
        g0 = _FLAG_BYTES
        r0 = g0 + rows_total * hidden * 2
        self.gather = raw[g0:r0].view(torch.bfloat16).view(rows_total, hidden)
        self.recv = raw[r0:].view(torch.bfloat16).view(world, self.R, hidden)
        self._g0, self._r0 = g0, r0
        self.e_gather = self.e_recv = self.e_barrier = 0    # epochs (every rank advances them identically)
        self.tiles_per_pass = (self.R // 128) * ((hidden + 255) // 256) * 8   # arrivals per source and o_proj pass
        self.push_ctas = _lib.lib().vllm_tp_norm_ctas(self.R)                # arrivals per source and norm_push
        # where my pushes land on each peer
        self._gather_dst = _ptr_array([b + g0 + rank * self.R * hidden * 2 for b in self.base])
        self._recv_dst = _ptr_array([b + r0 + rank * self.R * hidden * 2 for b in self.base])
        self._gather_flags = _ptr_array([b + _GATHER_FLAG for b in self.base])
        self._recv_flags = _ptr_array([b + _RECV_FLAG for b in self.base])
        self._barrier_flags = _ptr_array([b + _BARRIER_FLAG for b in self.base])
        self._own = int(own_ptr)

    # ---- construction -------------------------------------------------------------------------------------
    @staticmethod
    def _alloc(nbytes):
        p = ctypes.c_void_p()
        _lib.check(_lib.lib().vllm_peer_alloc(ctypes.byref(p), nbytes), "vllm_peer_alloc")
        return p.value

    @classmethod
    def virtual(cls, world, rows_total, hidden, device="cuda"):
        """`world` ranks on ONE device (tests, single-GPU debugging): W allocations, cross-referenced tables."""
        dev = torch.device(device)
        with torch.cuda.device(dev):
            ptrs = [cls._alloc(exchange_bytes(rows_total, hidden, world)) for _ in range(world)]
        owner = _Allocations(ptrs, [], dev)
        return [cls(r, world, rows_total, hidden, dev, ptrs[r], ptrs, owner) for r in range(world)]

    @classmethod
    def from_process_group(cls, rows_total, hidden, device, group=None):
        """One rank per process: allocate, all-gather the IPC handles over torch.distributed, map the peers."""
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        dev = torch.device(device)
        L = _lib.lib()
        with torch.cuda.device(dev):
            own = cls._alloc(exchange_bytes(rows_total, hidden, world))
            hb = L.vllm_peer_handle_bytes()
            buf = ctypes.create_string_buffer(hb)
            _lib.check(L.vllm_peer_export(own, buf), "vllm_peer_export")
            handles = [None] * world
            dist.all_gather_object(handles, bytes(buf.raw), group=group)
            # the arrival counts of the protocol assume every rank launches the norm/push kernel with the same CTA
            # count (peer.cu: min(rows, 4 x SMs)); MIG / MPS SM limits would break that silently -- check it
            ctas = [None] * world
            dist.all_gather_object(ctas, int(L.vllm_tp_norm_ctas(rows_total // world)), group=group)
            if len(set(ctas)) != 1:
                raise RuntimeError(f"tensor-parallel ranks disagree on the norm/push CTA count {ctas}: "
                                   "the GPUs of the group expose different SM counts")
            ptrs, opened = [], []
            for j in range(world):
                if j == rank:
                    ptrs.append(own)
                    continue
                p = ctypes.c_void_p()
                _lib.check(L.vllm_peer_open(ctypes.create_string_buffer(handles[j], hb), ctypes.byref(p)),
                           "vllm_peer_open")
                ptrs.append(p.value)
                opened.append(p.value)
            dist.barrier(group=group)
        return cls(rank, world, rows_total, hidden, dev, own, ptrs, _Allocations([own], opened, dev))

    # ---- exchange steps (each enqueues one kernel on the current stream) ------------------------------------
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def barrier(self):
        """Arrive: every rank has finished reading the buffers of the previous forward before anybody overwrites
        them.  Arrive and wait are separate launches so a lock-step driver can interleave virtual ranks."""
        self.e_barrier += 1
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().vllm_tp_signal(self._barrier_flags, self.world, 1, self._stream()), "vllm_tp_signal")

    def barrier_wait(self):
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().vllm_tp_wait(self._own + _BARRIER_FLAG, self.e_barrier * self.world, self._stream()),
                       "vllm_tp_wait")

    def norm_push(self, x_local, weight, eps):
        """gather[j][rank rows] = RMSNorm(x_local) * weight on every rank j (the all-gather, fused into the norm)."""
        self._check_rows(x_local)
        self.e_gather += 1
        with torch.cuda.device(self.device), ops._Prof("tp_norm_push", 0.0, 2.0 * x_local.numel() * (1 + self.world)):
            rc = _lib.lib().vllm_tp_reduce_norm_bf16(None, 0, 0, x_local.data_ptr(), weight.data_ptr(), float(eps),
                                                     self._gather_dst, self.world, self.H, None, 0,
                                                     self._gather_flags, self.world, self.R, self.H, self._stream())
        _lib.check(rc, "vllm_tp_reduce_norm_bf16")

    def gathered(self):
        """Wait for every rank's rows of the current gather epoch; returns the [M, H] buffer (a view, not a copy)."""
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().vllm_tp_wait(self._own + _GATHER_FLAG, self.e_gather * self.world * self.push_ctas,
                                               self._stream()), "vllm_tp_wait")
        return self.gather

    def oproj_scatter(self, ctx, w_shard):
        """partial = ctx @ w_shard.T pushed tile by tile into the row owners' receive slot `rank` (reduce-scatter)."""
        if ctx.dim() != 2 or ctx.shape[0] != self.M or ctx.dtype != torch.bfloat16 or ctx.stride(1) != 1:
            raise RuntimeError("oproj_scatter: ctx must be bf16 [M, K_local]")
        if w_shard.shape != (self.H, ctx.shape[1]) or w_shard.dtype != torch.bfloat16 or w_shard.stride(1) != 1:
            raise RuntimeError("oproj_scatter: w_shard must be bf16 [H, K_local]")
        self.e_recv += 1
        K = ctx.shape[1]
        with torch.cuda.device(self.device), ops._Prof("gemm", 2.0 * self.M * self.H * K,
                                                       2.0 * (self.M * K + self.H * K + self.M * self.H)):
            rc = _lib.lib().vllm_gemm_bf16_scatter(ctx.data_ptr(), ctx.stride(0), w_shard.data_ptr(),
                                                   w_shard.stride(0), self._recv_dst, self._recv_flags, self.world,
                                                   self.R, self.H, self.H, K, self._stream())
        _lib.check(rc, "vllm_gemm_bf16_scatter")

    def reduce_norm(self, x_local, weight, eps):
        """x_local += sum of the W partial slots (in place); returns RMSNorm(x_local) * weight for the local rows."""
        self._check_rows(x_local)
        h = torch.empty_like(x_local)
        dst = _ptr_array([h.data_ptr()])
        with torch.cuda.device(self.device), ops._Prof("tp_reduce_norm", 0.0, 2.0 * x_local.numel() * (self.world + 3)):
            rc = _lib.lib().vllm_tp_reduce_norm_bf16(self.recv.data_ptr(), self.world, self.R * self.H,
                                                     x_local.data_ptr(), weight.data_ptr(), float(eps), dst, 1, self.H,
                                                     self._own + _RECV_FLAG,
                                                     self.e_recv * self.world * self.tiles_per_pass, None, 0,
                                                     self.R, self.H, self._stream())
        _lib.check(rc, "vllm_tp_reduce_norm_bf16")
        return h

    def _check_rows(self, x):
        if x.shape != (self.R, self.H) or x.dtype != torch.bfloat16 or not x.is_contiguous():
            raise RuntimeError(f"expected contiguous bf16 [{self.R}, {self.H}] local rows")


class _Allocations:
    """Frees the cudaMalloc'ed exchange buffers / closes the IPC mappings when the last PeerComm goes away."""

    def __init__(self, owned, opened, device):
        self.owned, self.opened, self.device = list(owned), list(opened), device

    def __del__(self):
        try:
            L = _lib.lib()
            with torch.cuda.device(self.device):
                torch.cuda.synchronize()
                for p in self.opened:
                    L.vllm_peer_close(p)
                for p in self.owned:
                    L.vllm_peer_free(p)
        except Exception:
            pass


def shard_llama_state_dict(sd, config, rank, world):
    """HF-named full state dict -> the tensors rank `rank` holds: packed QKV rows of its heads, o_proj columns of its
    heads, everything else replicated (gate/up row-interleaved for the SwiGLU epilogue, like llama.LlamaMLP)."""
    nq = config.num_attention_heads
    nkv = getattr(config, "num_key_value_heads", None) or nq
    D = getattr(config, "head_dim", None) or config.hidden_size // nq
    if nq % world or nkv % world:
        raise ValueError(f"heads ({nq} q / {nkv} kv) must divide over {world} ranks")
    ql, kl = nq // world * D, nkv // world * D
    out = {"embed": sd["model.embed_tokens.weight"], "final_norm": sd["model.norm.weight"],
           "lm_head": sd["lm_head.weight"], "layers": []}
    for i in range(config.num_hidden_layers):
        p = f"model.layers.{i}."
        g, u = sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]
        out["layers"].append({
            "wqkv": torch.cat([sd[p + "self_attn.q_proj.weight"][rank * ql:(rank + 1) * ql],
                               sd[p + "self_attn.k_proj.weight"][rank * kl:(rank + 1) * kl],
                               sd[p + "self_attn.v_proj.weight"][rank * kl:(rank + 1) * kl]], 0).contiguous(),
            "wo": sd[p + "self_attn.o_proj.weight"][:, rank * ql:(rank + 1) * ql].contiguous(),
            "w_gate_up": torch.stack([g, u], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous(),
            "w_down": sd[p + "mlp.down_proj.weight"],
            "ln1": sd[p + "input_layernorm.weight"], "ln2": sd[p + "post_attention_layernorm.weight"],
        })
    return out


def shard_internlm2_state_dict(sd, config, rank, world):
    """The same shards from the reference's InternLM2 names (internlm2/modeling_internlm2.py: model.tok_embeddings,
    layers.N.attention.{wqkv,wo}, feed_forward.{w1,w2,w3}, attention_norm, ffn_norm, model.norm, output) -- the 26B
    preset's LLM.  `wqkv` interleaves, per KV head, (G query heads, k, v) along its rows (:337-349): rank r takes KV
    heads [r*nkv/W, (r+1)*nkv/W) WITH their G query heads each, so grouped-query attention stays rank-local and the
    rank's query heads are the contiguous global heads [r*nq/W, (r+1)*nq/W) that `wo`'s columns are ordered by."""
    nq = config.num_attention_heads
    nkv = getattr(config, "num_key_value_heads", None) or nq
    D = config.hidden_size // nq
    if nq % world or nkv % world:
        raise ValueError(f"heads ({nq} q / {nkv} kv) must divide over {world} ranks")
    if getattr(config, "bias", False):
        raise NotImplementedError("TP path: InternLM2 with projection biases")
    G, kvl = nq // nkv, nkv // world
    ql = kvl * G * D
    out = {"embed": sd["model.tok_embeddings.weight"], "final_norm": sd["model.norm.weight"],
           "lm_head": sd["output.weight"], "layers": []}
    for i in range(config.num_hidden_layers):
        p = f"model.layers.{i}."
        w = sd[p + "attention.wqkv.weight"]
        blk = w.view(nkv, G + 2, D, w.shape[1])[rank * kvl:(rank + 1) * kvl]           # this rank's KV-head groups
        g, u = sd[p + "feed_forward.w1.weight"], sd[p + "feed_forward.w3.weight"]
        out["layers"].append({
            "wqkv": torch.cat([blk[:, :G].reshape(-1, w.shape[1]), blk[:, G].reshape(-1, w.shape[1]),
                               blk[:, G + 1].reshape(-1, w.shape[1])], 0).contiguous(),
            "wo": sd[p + "attention.wo.weight"][:, rank * ql:(rank + 1) * ql].contiguous(),
            "w_gate_up": torch.stack([g, u], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous(),
            "w_down": sd[p + "feed_forward.w2.weight"],
            "ln1": sd[p + "attention_norm.weight"], "ln2": sd[p + "ffn_norm.weight"],
        })
    return out


class TPLlamaForCausalLM(nn.Module):
    """One rank of the tensor-parallel `B200LlamaForCausalLM`.  `comm` is a `PeerComm` (or, in CPU tests, a double
    with the same five methods)."""

    def __init__(self, config, comm, shards=None, device=None, dtype=torch.bfloat16):
        super().__init__()
        self.config, self.comm = config, comm
        self.nq = config.num_attention_heads
        self.nkv = getattr(config, "num_key_value_heads", None) or self.nq
        self.D = getattr(config, "head_dim", None) or config.hidden_size // self.nq
        W = comm.world
        if self.nq % W or self.nkv % W:
            raise ValueError(f"heads ({self.nq} q / {self.nkv} kv) must divide over {W} ranks")
        if getattr(config, "attention_bias", False) or getattr(config, "bias", False):
            raise NotImplementedError("TP path: projection biases")
        self.eps = config.rms_norm_eps
        theta = getattr(config, "rope_theta", None)
        if theta is None:
            rp = getattr(config, "rope_parameters", None) or {}
            theta = rp.get("rope_theta", 10000.0) if isinstance(rp, dict) else 10000.0
        self.theta = theta
        self.shards = None
        # forward_pipelined: optional SM budgets of the compute GEMMs / of the scatter GEMM (0 = all SMs, the default).
        # Not measured on H100s: the scatter GEMM's peer stores need many SMs to fill the links, so a budget may lose.
        self.compute_sms, self.scatter_sms = 0, 0
        if shards is not None:
            self.load_shards(shards, device, dtype)

    def load_shards(self, shards, device=None, dtype=torch.bfloat16):
        mv = (lambda t: t.detach().to(device=device, dtype=dtype).contiguous())
        self.shards = {k: (mv(v) if k != "layers" else [{n: mv(t) for n, t in lyr.items()} for lyr in v])
                       for k, v in shards.items()}
        return self

    @classmethod
    def from_full_state_dict(cls, config, comm, sd, device=None, dtype=torch.bfloat16):
        """HF Llama names (Vicuna, 7B preset) or the reference's InternLM2 names (26B preset), told apart by the keys."""
        shard = shard_internlm2_state_dict if "model.tok_embeddings.weight" in sd else shard_llama_state_dict
        return cls(config, comm, shard(sd, config, comm.rank, comm.world), device, dtype)

    @classmethod
    def random_init(cls, config, comm, device, seed=0, std=0.02):
        """Random shards without ever materialising the full model (bench: 7B at TP=8).  Replicated tensors use the
        same seed on every rank; sharded ones a rank-specific seed (they only have to be random)."""
        g = torch.Generator(device=device).manual_seed(seed)
        gr = torch.Generator(device=device).manual_seed(seed * 1000 + 17 + comm.rank)
        H, I, V = config.hidden_size, config.intermediate_size, config.vocab_size
        W = comm.world
        nq = config.num_attention_heads
        nkv = getattr(config, "num_key_value_heads", None) or nq
        D = getattr(config, "head_dim", None) or H // nq
        rn = lambda shape, gen: (torch.randn(shape, generator=gen, device=device, dtype=torch.float32) * std).to(torch.bfloat16)  # noqa: E731
        shards = {"embed": rn((V, H), g), "final_norm": torch.ones(H, device=device, dtype=torch.bfloat16),
                  "lm_head": rn((V, H), g), "layers": []}
        for _ in range(config.num_hidden_layers):
            shards["layers"].append({
                "wqkv": rn(((nq + 2 * nkv) // W * D, H), gr), "wo": rn((H, nq // W * D), gr),
                "w_gate_up": rn((2 * I, H), g), "w_down": rn((H, I), g),
                "ln1": torch.ones(H, device=device, dtype=torch.bfloat16),
                "ln2": torch.ones(H, device=device, dtype=torch.bfloat16)})
        m = cls(config, comm)
        m.shards = shards
        return m

    # ---- forward --------------------------------------------------------------------------------------------
    def phases(self, inputs_embeds, attention_mask=None, position_ids=None, compute_logits=True, comm=None, slot=None):
        """Generator: yields after every step that publishes data to peers, so `run_lockstep` can interleave the
        virtual ranks of one device.  The result is left in `self.result` (or `self.results[slot]` for a micro-batch
        of `forward_pipelined`, which passes that micro-batch's own `comm`)."""
        c, S = comm or self.comm, self.shards
        B, T, H = inputs_embeds.shape
        M = B * T
        if M != c.M or H != c.H:
            raise RuntimeError(f"comm was set up for [{c.M}, {c.H}] rows, got [{M}, {H}]")
        W, R, r = c.world, c.R, c.rank
        nql, nkvl, D = self.nq // W, self.nkv // W, self.D
        dev = inputs_embeds.device
        seqlens = right_padding_lengths(attention_mask)
        if position_ids is None:
            position_ids = torch.arange(T, device=dev)[None].expand(B, T)
        cos, sin = rope_tables(position_ids, D, self.theta, inputs_embeds.dtype)
        x = inputs_embeds.reshape(M, H)[r * R:(r + 1) * R].contiguous().clone()     # my rows of the residual stream
        c.barrier()
        yield "barrier"
        c.barrier_wait()
        c.norm_push(x, S["layers"][0]["ln1"], self.eps)
        yield "push"
        n_layers = len(S["layers"])
        for i, ly in enumerate(S["layers"]):
            hN = c.gathered()                                                         # [M, H], all tokens
            qkv = ops.linear(hN, ly["wqkv"])                                          # [M, (nql + 2 nkvl) D]
            ops.rope_(qkv, cos, sin, nql + nkvl, D)
            q = qkv[:, :nql * D].view(B, T, nql, D)
            k = qkv[:, nql * D:(nql + nkvl) * D].view(B, T, nkvl, D)
            v = qkv[:, (nql + nkvl) * D:].view(B, T, nkvl, D)
            ctx = ops.attention(q, k, v, causal=True, seqlens=seqlens)
            c.oproj_scatter(ctx.reshape(M, nql * D), ly["wo"])
            yield "scatter"
            h = c.reduce_norm(x, ly["ln2"], self.eps)                                 # x += sum partials; h = norm2(x)
            mid = ops.linear(h, ly["w_gate_up"], act="swiglu")
            x = ops.linear(mid, ly["w_down"], residual=x)
            nxt = S["layers"][i + 1]["ln1"] if i + 1 < n_layers else S["final_norm"]
            c.norm_push(x, nxt, self.eps)
            yield "push"
        last = c.gathered().clone().view(B, T, H)                                     # final-norm'ed states, all tokens
        logits = None
        if compute_logits:
            V = self.config.vocab_size
            Vp = (V + 3) // 4 * 4
            buf = torch.empty((R, Vp), dtype=torch.float32, device=dev)
            ops.linear(last.view(M, H)[r * R:(r + 1) * R], S["lm_head"], out=buf[:, :V])
            logits = buf[:, :V]
        # `hidden_states[-1]` / `logits` are what the composite forward reads (modeling_visionllmv2.py:733-751); the full
        # [B, T, V] logits are never materialised here -- each rank keeps the rows it owns.
        res = SimpleNamespace(last_hidden_state=last, hidden_states=(last,), logits=None, logits_local=logits,
                              row_range=(r * R, (r + 1) * R), past_key_values=None, attentions=None)
        if slot is None:
            self.result = res
        else:
            self.results[slot] = res

    # ---- micro-batch pipelining (r2): hide the layer's all-gather / reduce-scatter behind the other half's GEMMs ----------
    def micro_generators(self, micro_comms, inputs_embeds, attention_mask=None, position_ids=None, compute_logits=True):
        """One `phases` generator per micro-batch: the batch is cut into len(micro_comms) equal groups of sequences, each
        with its OWN exchange buffers / counters (`micro_comms[i]` is a PeerComm for B/n * T token rows), so the groups'
        protocols are independent and their kernels may overlap freely."""
        n = len(micro_comms)
        B = inputs_embeds.shape[0]
        if B % n:
            raise RuntimeError(f"batch {B} does not split into {n} micro-batches")
        b = B // n
        self.results = [None] * n
        cut = lambda t, i: None if t is None else t[i * b:(i + 1) * b]   # noqa: E731
        return [self.phases(cut(inputs_embeds, i), cut(attention_mask, i), cut(position_ids, i), compute_logits,
                            comm=micro_comms[i], slot=i) for i in range(n)]

    @torch.no_grad()
    def forward_pipelined(self, micro_comms, inputs_embeds=None, input_ids=None, attention_mask=None, position_ids=None,
                          compute_logits=True):
        """The same forward with the batch cut into micro-batches that run on their own CUDA streams: while one
        micro-batch waits for its peers' o_proj partials or pushes its normalised rows over NVLink (both bound by the
        link, not by the SMs), the other one's GEMMs own the tensor cores.  Results: `last_hidden_state` of the whole
        batch; `logits_local` / `row_range` become per-micro-batch lists (a rank owns R / n rows of every micro-batch)."""
        if inputs_embeds is None:
            inputs_embeds = torch.nn.functional.embedding(input_ids, self.shards["embed"])
        dev = inputs_embeds.device
        n = len(micro_comms)
        if getattr(self, "_streams", None) is None or len(self._streams) != n:
            self._streams = [torch.cuda.Stream(device=dev) for _ in range(n)]
        main = torch.cuda.current_stream(dev)
        gens = self.micro_generators(micro_comms, inputs_embeds, attention_mask, position_ids, compute_logits)
        for st in self._streams:
            st.wait_stream(main)
        # a GEMM CTA owns its SM (register file), so the other micro-batch's link-bound steps overlap a GEMM only on SMs
        # its grid leaves free: compute GEMMs get `compute_sms`, the scatter GEMM (NVLink-bound epilogue) `scatter_sms`
        n_sms = torch.cuda.get_device_properties(dev).multi_processor_count
        comp = int(os.environ.get("VLLM_TP_COMPUTE_SMS", self.compute_sms))
        scat = int(os.environ.get("VLLM_TP_SCATTER_SMS", self.scatter_sms))
        if micro_comms[0].world > 1 and 0 < comp < n_sms:
            _lib.check(_lib.lib().vllm_gemm_set_sm_limit(comp, scat), "vllm_gemm_set_sm_limit")
        try:
            live = True
            while live:                                    # round-robin issue: the streams' kernels interleave on the device
                live = False
                for g, st in zip(gens, self._streams):
                    with torch.cuda.stream(st):
                        try:
                            next(g)
                            live = True
                        except StopIteration:
                            pass
        finally:
            _lib.lib().vllm_gemm_set_sm_limit(0, 0)
        for st, res in zip(self._streams, self.results):
            main.wait_stream(st)
            res.last_hidden_state.record_stream(main)
            if res.logits_local is not None:
                res.logits_local.record_stream(main)
        last = torch.cat([r.last_hidden_state for r in self.results], 0)
        self.result = SimpleNamespace(last_hidden_state=last, hidden_states=(last,), logits=None,
                                      logits_local=[r.logits_local for r in self.results],
                                      row_range=[r.row_range for r in self.results], past_key_values=None, attentions=None)
        return self.result

    # ---- the parts of the HF interface the composite model touches (modeling_visionllmv2.py:420,571,724-751) -------
    @property
    def dtype(self):
        return self.shards["lm_head"].dtype

    def get_input_embeddings(self):
        return lambda ids: torch.nn.functional.embedding(ids, self.shards["embed"])

    @torch.no_grad()
    def forward(self, inputs_embeds=None, input_ids=None, attention_mask=None, position_ids=None,
                compute_logits=True, past_key_values=None, use_cache=False, output_attentions=False,
                output_hidden_states=True, return_dict=True):
        if past_key_values is not None or use_cache:
            raise NotImplementedError("KV-cache decoding is outside the forward hot path (SURVEY 3.4)")
        if inputs_embeds is None:
            inputs_embeds = torch.nn.functional.embedding(input_ids, self.shards["embed"])
        for _ in self.phases(inputs_embeds, attention_mask, position_ids, compute_logits):
            pass
        return self.result


@torch.no_grad()
def run_lockstep_micro(ranks, micro_comms_per_rank, inputs_embeds, **kw):
    """`run_lockstep` for the micro-batched forward: every (virtual rank, micro-batch) generator advances phase by phase
    on the current stream.  Returns per-rank lists of per-micro-batch results."""
    gens = [g for m, mc in zip(ranks, micro_comms_per_rank) for g in m.micro_generators(mc, inputs_embeds, **kw)]
    live = True
    while live:
        live = False
        for g in gens:
            try:
                next(g)
                live = True
            except StopIteration:
                pass
    return [m.results for m in ranks]


@torch.no_grad()
def run_lockstep(ranks, inputs_embeds, **kw):
    """Advance the forwards of several (virtual) ranks phase by phase on the current stream: every rank publishes
    before any rank consumes, so no wait kernel ever spins.  Returns the per-rank results."""
    gens = [m.phases(inputs_embeds, **kw) for m in ranks]
    live = True
    while live:
        live = False
        for g in gens:
            try:
                next(g)
                live = True
            except StopIteration:
                pass
    return [m.result for m in ranks]
