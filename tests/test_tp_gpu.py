"""GPU: the tensor-parallel Llama path (visionllm_b200/tp.py, csrc/peer.cu, vllm_gemm_bf16_scatter).

* kernel-level: the scatter GEMM (row blocks -> per-destination slots + arrival counts) and the fused
  reduce + residual + RMSNorm + push kernel against fp32 torch on the same bf16 inputs;
* protocol-level on ONE device: W = 2 / 4 virtual ranks advanced in lock step (PeerComm.virtual + run_lockstep) --
  pointer tables, receive slots, gather buffer, counters and epochs exactly as in the multi-process run -- compared
  with the unsharded `B200LlamaForCausalLM` and with HF `LlamaForCausalLM` (fp32 and bf16, the module tolerance rule of
  test_modules_gpu.py), twice in a row (epoch counters);
* multi-process over CUDA IPC + NVLink when the machine has >= 2 GPUs (skipped otherwise).
"""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_l2(a, b):
    return float(torch.linalg.norm(a.float() - b.float()) / torch.linalg.norm(b.float()))


def _flag(comm, off):
    from visionllm_b200.tp import _DeviceBytes
    raw = torch.as_tensor(_DeviceBytes(comm._own, 4096), device="cuda")
    return int(raw[off:off + 4].view(torch.int32).item())


@pytest.mark.parametrize("K", [128, 1024])          # short and long K
def test_scatter_gemm_fills_owner_slots(K):
    from visionllm_b200 import tp
    W, M, H = 2, 512, 320                            # H % 256 != 0: ragged last column tile
    comms = tp.PeerComm.virtual(W, M, H)
    g = torch.Generator(device="cuda").manual_seed(0)
    ctxs = [torch.randn(M, K, generator=g, device="cuda").bfloat16() for _ in range(W)]
    ws = [(torch.randn(H, K, generator=g, device="cuda") * 0.1).bfloat16() for _ in range(W)]
    for c, a, w in zip(comms, ctxs, ws):
        c.oproj_scatter(a, w)
    torch.cuda.synchronize()
    R = M // W
    for d, c in enumerate(comms):
        assert _flag(c, tp._RECV_FLAG) == W * c.tiles_per_pass
        for s in range(W):
            want = (ctxs[s].float() @ ws[s].float().T)[d * R:(d + 1) * R]
            got = c.recv[s].float()
            assert (got - want).abs().max() <= 2 ** -8 * want.abs().max() + 1e-6


def test_reduce_norm_kernel_matches_fp32():
    from visionllm_b200 import tp
    W, M, H = 4, 1024, 4096
    comms = tp.PeerComm.virtual(W, M, H)
    c = comms[1]
    g = torch.Generator(device="cuda").manual_seed(1)
    c.recv.copy_(torch.randn(W, c.R, H, generator=g, device="cuda"))
    x = torch.randn(c.R, H, generator=g, device="cuda").bfloat16()
    w = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).bfloat16()
    x0 = x.clone()
    c.e_recv = 0                                      # target 0: no wait
    h = c.reduce_norm(x, w, 1e-5)
    acc = torch.zeros(c.R, H, device="cuda")
    for s_ in range(W):                               # the kernel's order: slots 0..W-1, then the residual
        acc += c.recv[s_].float()
    xs = (acc + x0.float()).bfloat16()
    assert torch.equal(x, xs)                         # one bf16 rounding of the fp32 sum
    xf = xs.float()
    hn = (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).bfloat16().float()).bfloat16()
    assert (h.float() - hn.float()).abs().max() <= 2 ** -7 * hn.float().abs().max()
    assert rel_l2(h, hn) < 2e-3
    # push form: every peer's gather rows + counters
    c.norm_push(x, w, 1e-5)
    torch.cuda.synchronize()
    for d in comms:
        assert torch.equal(d.gather[c.rank * c.R:(c.rank + 1) * c.R], h)
        assert _flag(d, tp._GATHER_FLAG) == c.push_ctas


def _tiny_cfg():
    from transformers import LlamaConfig
    return LlamaConfig(hidden_size=512, intermediate_size=1376, num_hidden_layers=2, num_attention_heads=4,
                       num_key_value_heads=4, vocab_size=1000, rms_norm_eps=1e-5, max_position_embeddings=512,
                       attn_implementation="eager")


def _hf_and_inputs(padded):
    from transformers import LlamaForCausalLM
    cfg = _tiny_cfg()
    torch.manual_seed(0)
    hf = LlamaForCausalLM(cfg).eval()
    sd = {k: v.to(torch.bfloat16).float() for k, v in hf.state_dict().items()}
    hf.load_state_dict(sd)
    B, T = 2, 256
    emb = (torch.randn(B, T, 512, generator=torch.Generator().manual_seed(1)) * 0.5).bfloat16()
    am = torch.ones(B, T, dtype=torch.long)
    if padded:
        am[1, 200:] = 0
    return cfg, hf, sd, emb, am


@pytest.mark.parametrize("world,padded", [(2, False), (4, True)])
def test_tp_virtual_ranks_match_unsharded(world, padded):
    from visionllm_b200 import tp
    from visionllm_b200.llama import B200LlamaForCausalLM
    cfg, hf, sd, emb, am = _hf_and_inputs(padded)
    B, T, H = emb.shape
    with torch.no_grad():
        ref32 = hf.float().cuda()(inputs_embeds=emb.float().cuda(), attention_mask=am.cuda(), output_hidden_states=True)
        ref16 = hf.bfloat16()(inputs_embeds=emb.cuda(), attention_mask=am.cuda(), output_hidden_states=True)
    single = B200LlamaForCausalLM(cfg)
    single.load_state_dict(sd, strict=True)
    single = single.to("cuda", torch.bfloat16).eval()
    one = single(inputs_embeds=emb.cuda(), attention_mask=am.cuda(), output_hidden_states=True)
    comms = tp.PeerComm.virtual(world, B * T, H)
    ranks = [tp.TPLlamaForCausalLM.from_full_state_dict(cfg, c, sd, device="cuda") for c in comms]
    valid = am.bool().cuda().reshape(-1)
    for rep in range(2):                               # second pass: epochs advance, buffers are reused
        res = tp.run_lockstep(ranks, emb.cuda(), attention_mask=am.cuda())
        torch.cuda.synchronize()
        logits = torch.cat([r.logits_local for r in res], 0)
        assert [r.row_range for r in res] == [(i * B * T // world, (i + 1) * B * T // world) for i in range(world)]
        for r in res:                                  # every rank holds the same gathered final states
            assert torch.equal(r.last_hidden_state, res[0].last_hidden_state)
        hs = res[0].last_hidden_state.reshape(B * T, H)[valid]
        r32h, r16h = ref32.hidden_states[-1].reshape(B * T, H)[valid], ref16.hidden_states[-1].reshape(B * T, H)[valid]
        assert rel_l2(hs, r32h) <= 1.5 * rel_l2(r16h, r32h) + 1e-3, (rel_l2(hs, r32h), rel_l2(r16h, r32h))
        r32l, r16l = ref32.logits.reshape(B * T, -1)[valid], ref16.logits.reshape(B * T, -1)[valid]
        assert rel_l2(logits[valid], r32l) <= 1.5 * rel_l2(r16l, r32l) + 1e-3
        # vs our own unsharded path: differs only by the bf16 rounding of the W o_proj partials
        assert rel_l2(hs, one.hidden_states[-1].reshape(B * T, H)[valid]) < 1e-2
    assert logits.dtype == torch.float32 and logits.shape == (B * T, 1000)


def test_tp_world1_matches_unsharded():
    """W = 1: the scatter GEMM, the reduce kernel (one slot) and the push kernel must reproduce the plain path up to
    the extra bf16 rounding of the single o_proj 'partial'."""
    from visionllm_b200 import tp
    from visionllm_b200.llama import B200LlamaForCausalLM
    cfg, hf, sd, emb, am = _hf_and_inputs(False)
    B, T, H = emb.shape
    single = B200LlamaForCausalLM(cfg)
    single.load_state_dict(sd, strict=True)
    single = single.to("cuda", torch.bfloat16).eval()
    one = single(inputs_embeds=emb.cuda(), output_hidden_states=True)
    comm = tp.PeerComm.virtual(1, B * T, H)[0]
    m = tp.TPLlamaForCausalLM.from_full_state_dict(cfg, comm, sd, device="cuda")
    out = m(inputs_embeds=emb.cuda())
    assert rel_l2(out.last_hidden_state, one.hidden_states[-1]) < 5e-3
    assert rel_l2(out.logits_local.view(B, T, -1), one.logits) < 5e-3


@pytest.mark.parametrize("world", [1, 2])
def test_tp_micro_batched_forward_equals_the_plain_forward(world):
    """r2: the batch cut into two micro-batches with their own exchange buffers (TPLlamaForCausalLM.micro_generators /
    forward_pipelined: two CUDA streams, the halves' exchange steps hide behind each other's GEMMs) must give the plain
    forward's states and logits -- every op is row-wise or per sequence.  W = 1 runs the real two-stream schedule, W = 2
    the virtual ranks in lock step; twice in a row (epochs, buffer reuse)."""
    from visionllm_b200 import tp
    cfg, hf, sd, emb, am = _hf_and_inputs(False)
    B, T, H = emb.shape
    assert B % 2 == 0
    comms = tp.PeerComm.virtual(world, B * T, H)
    ranks = [tp.TPLlamaForCausalLM.from_full_state_dict(cfg, c, sd, device="cuda") for c in comms]
    plain = tp.run_lockstep(ranks, emb.cuda())
    torch.cuda.synchronize()
    micro = [tp.PeerComm.virtual(world, B * T // 2, H) for _ in range(2)]          # micro[i][rank]
    per_rank = [[micro[i][r] for i in range(2)] for r in range(world)]
    Rm = B * T // 2 // world
    for rep in range(2):
        if world == 1:
            out = ranks[0].forward_pipelined(per_rank[0], inputs_embeds=emb.cuda())
            torch.cuda.synchronize()
            res = [ranks[0].results]
            assert torch.equal(out.last_hidden_state, plain[0].last_hidden_state)
        else:
            res = tp.run_lockstep_micro(ranks, per_rank, emb.cuda())
            torch.cuda.synchronize()
        full_logits = torch.cat([p.logits_local for p in plain], 0).view(B, T, -1)
        for r in range(world):
            for i in range(2):
                got = res[r][i]
                assert torch.equal(got.last_hidden_state, plain[0].last_hidden_state[i * (B // 2):(i + 1) * (B // 2)])
                assert got.row_range == (r * Rm, (r + 1) * Rm)
                want = full_logits[i * (B // 2):(i + 1) * (B // 2)].reshape(B * T // 2, -1)[r * Rm:(r + 1) * Rm]
                assert torch.equal(got.logits_local, want)


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["VLLM_ROOT"])
from visionllm_b200 import tp
from visionllm_b200.llama import B200LlamaForCausalLM
from transformers import LlamaConfig, LlamaForCausalLM
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
cfg = LlamaConfig(hidden_size=512, intermediate_size=1376, num_hidden_layers=3, num_attention_heads=4,
                  num_key_value_heads=4, vocab_size=1000, rms_norm_eps=1e-5, max_position_embeddings=512)
torch.manual_seed(0)
sd = {k: v.to(torch.bfloat16).float() for k, v in LlamaForCausalLM(cfg).state_dict().items()}
B, T, H = 2, 256, 512
emb = (torch.randn(B, T, H, generator=torch.Generator().manual_seed(1)) * 0.5).bfloat16().cuda()
single = B200LlamaForCausalLM(cfg); single.load_state_dict(sd); single = single.to("cuda", torch.bfloat16).eval()
one = single(inputs_embeds=emb, output_hidden_states=True)
comm = tp.PeerComm.from_process_group(B * T, H, torch.device("cuda", rank))
m = tp.TPLlamaForCausalLM.from_full_state_dict(cfg, comm, sd, device="cuda")
rel = lambda a, b: float(torch.linalg.norm(a.float() - b.float()) / torch.linalg.norm(b.float()))
for rep in range(3):
    out = m(inputs_embeds=emb)
    torch.cuda.synchronize()
    lo, hi = out.row_range
    e1 = rel(out.last_hidden_state, one.hidden_states[-1])
    e2 = rel(out.logits_local, one.logits.reshape(B * T, -1)[lo:hi])
    assert e1 < 1e-2 and e2 < 1e-2, (rank, rep, e1, e2)
mc = [tp.PeerComm.from_process_group(B * T // 2, H, torch.device("cuda", rank)) for _ in range(2)]
for rep in range(3):
    outp = m.forward_pipelined(mc, inputs_embeds=emb)
    torch.cuda.synchronize()
    assert torch.equal(outp.last_hidden_state, out.last_hidden_state), (rank, rep, "pipelined states differ")
dist.barrier()
print(f"rank {rank} ok {e1:.2e} {e2:.2e}", flush=True)
dist.destroy_process_group()
"""


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp_two_processes_over_ipc(tmp_path):
    script = tmp_path / "tp_worker.py"
    script.write_text(_WORKER)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    env = dict(os.environ, VLLM_ROOT=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "rank 0 ok" in r.stdout and "rank 1 ok" in r.stdout
