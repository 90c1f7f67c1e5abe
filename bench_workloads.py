"""Workloads for bench.py (measurement infrastructure, not product code).

Each workload is one pass of (a part of) the hot path over one batch of
synthetic input (SURVEY.md 8d).  `step_device` runs with inputs resident in
HBM; `step_e2e` goes through the same public API with HOST (pinned) buffers,
host<->device copies inside the timed region.
"""
import json
import os
import time

ROOT = os.path.dirname(os.path.abspath(__file__))


def measured_peaks():
    """Roofline denominators: NVIDIA's data sheet for the H100 SXM (3.35 TB/s HBM3; 989 TFLOP/s dense bf16 at up to
    700 W).  Data-sheet figures, not measurements: a power-limited card sustains less."""
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "H100 SXM data sheet"}


def gpu_identity(index):
    """Name and power limit of CUDA device `index` (they are part of every absolute number).  nvidia-smi is asked by the
    device's UUID: its own indices ignore CUDA_VISIBLE_DEVICES."""
    import subprocess
    import torch
    props = torch.cuda.get_device_properties(index)
    ident = {"name": props.name, "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", f"GPU-{props.uuid}"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        ident["power_limit_w"] = float(out)
    except Exception:
        pass
    return ident


def output_arrays(out, prefix="out"):
    """(name, tensor) for every tensor a caller of the timed path receives: a tensor, or tensors nested in tuples / lists /
    dicts / output objects (attributes), in a fixed order; None and non-tensor leaves are skipped."""
    import torch
    if isinstance(out, torch.Tensor):
        return [(prefix, out)]
    if isinstance(out, dict):
        items = [(str(k), v) for k, v in out.items()]
    elif isinstance(out, (tuple, list)):
        items = [(str(i), v) for i, v in enumerate(out)]
    elif hasattr(out, "__dict__"):
        items = sorted(vars(out).items())
    else:
        return []
    return [pair for k, v in items for pair in output_arrays(v, f"{prefix}.{k}")]


DUMP_BUDGET_BYTES = 60 * 1000 * 1000       # payload; the .npy headers (128 B each) stay far inside 64 MB (decimal) with it


def dump_outputs(out, directory, budget_bytes=DUMP_BUDGET_BYTES):
    """DIR/<name>.npy for every output tensor: float32 (float64 for 8-byte types), whole when it fits its equal share of
    the budget, else every k-th element of the flattened tensor starting at a seeded offset below k (distinct positions,
    the same on every run)."""
    import numpy as np
    import torch
    arrays = output_arrays(out)
    if not arrays:
        raise RuntimeError("the workload's last step left no output tensors to dump")
    os.makedirs(directory, exist_ok=True)
    share = budget_bytes // len(arrays)
    offsets = np.random.default_rng(0)
    for name, t in arrays:
        t = t.detach()
        wide = t.dtype in (torch.float64, torch.int64)
        keep = max(1, share // (8 if wide else 4))
        if t.numel() > keep:
            step = -(-t.numel() // keep)
            t = t.reshape(-1)[int(offsets.integers(0, step))::step]
        np.save(os.path.join(directory, name + ".npy"), t.to(torch.float64 if wide else torch.float32).cpu().numpy())


def shard_range(total, rank, world):
    """Contiguous batch shard of SURVEY 8e: rank r owns units [r*total/world, (r+1)*total/world)."""
    if total % world:
        raise ValueError(f"global batch {total} must divide over {world} ranks")
    per = total // world
    return rank * per, (rank + 1) * per


def max_over_ranks(value, dist=None, device="cpu"):
    """Multi-GPU timing rule: the step time of the job is the MAX over ranks (all_reduce MAX)."""
    import torch
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


GDINO_LEVELS_1024 = [(128, 128), (64, 64), (32, 32), (16, 16)]   # strides 8..64 of a 1024x1024 image


def msda_encoder_inputs(torch, N, device, seed, shapes_l=GDINO_LEVELS_1024, M=8, D=32, P=4, sigma=0.02):
    """SURVEY 8d cfg 2b 'enc': queries are the pixels, refs = pixel centres + N(0, sigma) offsets."""
    g = torch.Generator(device=device).manual_seed(seed)
    shapes = torch.tensor(shapes_l, dtype=torch.int64, device=device)
    L = len(shapes_l)
    S = sum(h * w for h, w in shapes_l)
    lsi = torch.cat((shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]))
    value = torch.randn(N, S, M, D, device=device, generator=g)
    refs = []
    for (H, W) in shapes_l:
        ys, xs = torch.meshgrid(torch.arange(H, device=device, dtype=torch.float32),
                                torch.arange(W, device=device, dtype=torch.float32), indexing="ij")
        refs.append(torch.stack(((xs + 0.5) / W, (ys + 0.5) / H), -1).reshape(-1, 2))
    ref_pts = torch.cat(refs, 0)[None, :, None, None, None, :]
    loc = (ref_pts + torch.randn(N, S, M, L, P, 2, device=device, generator=g) * sigma).contiguous()
    attw = torch.softmax(torch.randn(N, S, M, L * P, device=device, generator=g), -1).view(N, S, M, L, P)
    return value, shapes, lsi, loc, attw.contiguous()


class MsdaEncoderWorkload:
    """MSDA forward at the GDINO 1024^2 encoder shape (BASELINE cfg 2b): N=8, S=Lq=21760, M=8, D=32, L=4, P=4."""
    metric = "msda_encoder_layer_images_per_sec"
    unit = "images/s"
    dtype = "f32"
    N = 8

    def __init__(self, rank, world, device):
        self.rank, self.world, self.device = rank, world, device

    def setup(self):
        import torch
        import visionllm_b200.msda as ext
        self.torch, self.ext = torch, ext
        self.value, self.shapes, self.lsi, self.loc, self.attw = msda_encoder_inputs(
            torch, self.N, self.device, 1234 + self.rank)
        self.host_shapes = self.shapes.cpu()
        self.h_in = [t.cpu().pin_memory() for t in (self.value, self.loc, self.attw)]
        self.d_in = [torch.empty_like(t) for t in (self.value, self.loc, self.attw)]
        S = self.value.shape[1]
        self.h_out = torch.empty((self.N, S, 256), dtype=torch.float32).pin_memory()
        self.h2d_bytes = sum(t.numel() * 4 for t in self.h_in)
        self.d2h_bytes = self.h_out.numel() * 4
        # compulsory bytes per image (SURVEY 8d): value + loc + attw once, out once
        self.alg_bytes_per_image = (self.value[0].numel() + self.loc[0].numel() + self.attw[0].numel()
                                    + S * 256) * 4

    def step_device(self):
        self.out = self.ext.ms_deform_attn_forward(self.value, self.shapes, self.lsi, self.loc, self.attw, 64,
                                                   host_shapes=self.host_shapes)

    def step_e2e(self):
        for d, h in zip(self.d_in, self.h_in):
            d.copy_(h, non_blocking=True)
        out = self.ext.ms_deform_attn_forward(self.d_in[0], self.shapes, self.lsi, self.d_in[1], self.d_in[2], 64,
                                              host_shapes=self.host_shapes)
        self.h_out.copy_(out, non_blocking=True)

    def units_per_step(self):
        return self.N

    def dominant_kernel_ms(self, steps):
        torch = self.torch
        torch.cuda.synchronize()
        evs = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); self.step_device(); e1.record()
            evs.append((e0, e1))
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in evs) / steps

    def roofline(self, kern_ms, peaks):
        ach = self.alg_bytes_per_image * self.N / (kern_ms * 1e-3) / 1e9
        return {"kernel": "msda_fwd_warp_kernel", "bound": "hbm", "achieved": ach, "peak": peaks["hbm_gbs"],
                "peak_source": peaks["source"], "unit": "GB/s", "frac": ach / peaks["hbm_gbs"],
                "traffic": None, "kernel_ms": kern_ms,
                "algorithmic_bytes_per_launch": self.alg_bytes_per_image * self.N}

    def config(self):
        return {"workload": "msda_fwd encoder shape (BASELINE cfg 2b): N=8 S=Lq=21760 M=8 D=32 L=4 P=4 fp32",
                "l2_policy": "inputs_exceed_l2 (624 MB per step > 50 MB L2)", "parallelism": f"dp{self.world}"}

    def extra(self):
        return {}


class MsdaEncoderBf16Workload(MsdaEncoderWorkload):
    """cfg 2b "fast mode": value in bf16 (what the module's value_proj GEMM produces), sampling_loc / attn_weight fp32,
    fp32 accumulation, bf16 output -- `ms_deform_attn_forward_bf16`."""
    metric = "msda_encoder_layer_images_per_sec_bf16_value"
    dtype = "bf16 value/out, f32 locations, weights and accumulation"

    def setup(self):
        super().setup()
        torch = self.torch
        self.value = self.value.bfloat16()
        self.h_in = [t.cpu().pin_memory() for t in (self.value, self.loc, self.attw)]
        self.d_in = [torch.empty_like(t) for t in (self.value, self.loc, self.attw)]
        S = self.value.shape[1]
        self.h_out = torch.empty((self.N, S, 256), dtype=torch.bfloat16).pin_memory()
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in self.h_in)
        self.d2h_bytes = self.h_out.numel() * 2
        self.alg_bytes_per_image = (self.value[0].numel() * 2 + self.loc[0].numel() * 4 + self.attw[0].numel() * 4
                                    + S * 256 * 2)

    def step_device(self):
        self.out = self.ext.ms_deform_attn_forward_bf16(self.value, self.shapes, self.lsi, self.loc, self.attw)

    def step_e2e(self):
        for d, h in zip(self.d_in, self.h_in):
            d.copy_(h, non_blocking=True)
        out = self.ext.ms_deform_attn_forward_bf16(self.d_in[0], self.shapes, self.lsi, self.d_in[1], self.d_in[2])
        self.h_out.copy_(out, non_blocking=True)

    def config(self):
        c = super().config()
        c["workload"] = "msda_fwd encoder shape (BASELINE cfg 2b, fast mode): N=8 S=Lq=21760 M=8 D=32 L=4 P=4, bf16 value/out"
        c["l2_policy"] = "inputs_exceed_l2 (446 MB per step > 50 MB L2)"
        return c


class MsdaEncoderPairsWorkload(MsdaEncoderBf16Workload):
    """cfg 2b fast mode on the paired-row layout: a step = `ms_deform_attn_pack_pairs` (bf16 value -> [N,S,M,2,32], one
    HBM pass) + `ms_deform_attn_forward_pairs` (two 128-byte line fetches per sample instead of four); both launches
    are inside the timed region, the algorithmic bytes stay those of the bf16 operator (the pair tensor is internal)."""
    metric = "msda_encoder_layer_images_per_sec_bf16_value"

    def _run(self, value, loc, attw):
        pairs = self.ext.ms_deform_attn_pack_pairs(value, self.shapes, self.lsi)
        return self.ext.ms_deform_attn_forward_pairs(pairs, self.shapes, self.lsi, loc, attw)

    def step_device(self):
        self.out = self._run(self.value, self.loc, self.attw)

    def step_e2e(self):
        for d, h in zip(self.d_in, self.h_in):
            d.copy_(h, non_blocking=True)
        self.h_out.copy_(self._run(*self.d_in), non_blocking=True)

    def dominant_kernel_ms(self, steps):
        torch = self.torch
        pairs = self.ext.ms_deform_attn_pack_pairs(self.value, self.shapes, self.lsi)
        torch.cuda.synchronize()
        evs = []
        for _ in range(steps):
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            pairs = None                       # hand the block back first: no cudaMalloc inside the timed interval
            e0.record()
            pairs = self.ext.ms_deform_attn_pack_pairs(self.value, self.shapes, self.lsi)
            e1.record()
            self.ext.ms_deform_attn_forward_pairs(pairs, self.shapes, self.lsi, self.loc, self.attw)
            e2.record()
            evs.append((e0, e1, e2))
        torch.cuda.synchronize()
        self.pack_ms = sum(a.elapsed_time(b) for a, b, _ in evs) / steps
        self.gather_ms = sum(b.elapsed_time(c) for _, b, c in evs) / steps
        return self.pack_ms + self.gather_ms

    def roofline(self, kern_ms, peaks):
        r = super().roofline(kern_ms, peaks)
        r["kernel"] = "msda_pack_pairs_kernel + msda_fwd_pair_kernel (both launches of the step)"
        r["pack_ms"], r["gather_ms"] = self.pack_ms, self.gather_ms
        return r

    def config(self):
        c = super().config()
        c["workload"] += ", paired-row layout (pack + gather)"
        return c


def anyres_tiles_1024(torch, n_pairs, device, seed, tile=448, dtype=None, tiles=5):
    """What the reference's data pipeline hands to forward() for a 1024x1024 image under 'anyres'
    (mm_utils.py:39-75: image_size 448, max 6 tiles -> (2,2) grid + thumbnail = 5 tiles): a list of
    [5, 3, 448, 448] tensors, floats already cast to bf16 by dict_to_cuda (util/misc.py:499-515)."""
    g = torch.Generator(device=device).manual_seed(seed)
    return [torch.randn(tiles, 3, tile, tile, device=device, generator=g).to(dtype or torch.bfloat16)
            for _ in range(n_pairs)]


class PairForwardWorkload:
    """BASELINE cfg 3: VisionLLMv2 (InternViT-6B + Vicuna-7B), random init, bf16 forward of B (image, prompt)
    pairs per GPU: 5 anyres tiles of a 1024^2 image -> 48-layer ViT -> pixel shuffle -> internvl_mlp bridge ->
    1280 image tokens + 256 text tokens -> 32-layer LLM -> fp32 logits for every position."""
    metric = "img_text_pairs_per_sec_fwd_1024px_256tok"
    unit = "pairs/s"
    dtype = "bf16"
    PAIRS = 8
    IMP, VOCAB = 32002, 32026
    TILE, TOK_PER_TILE, TILES = 448, 256, 5            # anyres (2, 2) grid + thumbnail; 1024 ViT tokens -> pixel shuffle -> 256
    BRIDGE, PIXEL_SHUFFLE, VIS_LAYER = "internvl_mlp", True, -1
    vit = dict(hidden_size=3200, num_attention_heads=25, num_hidden_layers=48, intermediate_size=12800,
               image_size=448, patch_size=14)
    llm = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
               num_key_value_heads=32, vocab_size=VOCAB, rms_norm_eps=1e-5, max_position_embeddings=4096)

    def __init__(self, rank, world, device):
        self.rank, self.world, self.device = rank, world, device

    def build(self):
        import torch
        from types import SimpleNamespace
        from transformers import LlamaConfig
        from visionllm_b200.internvit import B200InternVisionModel, InternVisionConfig
        from visionllm_b200.llama import B200LlamaForCausalLM
        from visionllm_b200.modeling import B200VisionLLMv2Model
        cfg = SimpleNamespace(use_pixelshuffle=self.PIXEL_SHUFFLE, vl_bridge_type=self.BRIDGE, vis_output_layer=self.VIS_LAYER,
                              num_embs=4, imp_token_id=self.IMP, emb_token_id=32010, det_tool_id=32003, seg_tool_id=32005,
                              grd_tool_id=32004, pose_tool_id=32006)
        with torch.device("meta"):
            model = B200VisionLLMv2Model(cfg, self.vision_tower(), B200LlamaForCausalLM(LlamaConfig(**self.llm)))
        model = model.to_empty(device=self.device).to(torch.bfloat16)
        g = torch.Generator(device=self.device).manual_seed(0)      # same weights on every rank
        with torch.no_grad():
            for name, p in model.named_parameters():
                last = name.split(".")[-1]
                if "norm" in name and last == "weight":
                    p.fill_(1.0)
                elif last in ("ls1", "ls2"):
                    p.fill_(0.1)
                elif p.dim() <= 1:
                    p.zero_()
                else:
                    p.copy_(torch.randn(p.shape, device=self.device, generator=g, dtype=torch.float32) * 0.02)
        return model.eval()

    def vision_tower(self):
        from visionllm_b200.internvit import B200InternVisionModel, InternVisionConfig
        return B200InternVisionModel(InternVisionConfig(**self.vit))

    def setup(self):
        import torch
        self.torch = torch
        self.model = self.build()
        n_img = self.TILES * self.TOK_PER_TILE
        T = n_img + 256
        g = torch.Generator(device=self.device).manual_seed(1234 + self.rank)
        ids = torch.randint(0, 32000, (self.PAIRS, T), device=self.device, generator=g)
        ids[:, :n_img] = self.IMP
        self.ids = ids
        self.mask = torch.ones_like(ids)
        self.images = anyres_tiles_1024(torch, self.PAIRS, self.device, 99 + self.rank, tile=self.TILE, tiles=self.TILES)
        self.h_images = [t.cpu().pin_memory() for t in self.images]
        self.h_ids = ids.cpu().pin_memory()
        self.d_images = [torch.empty_like(t) for t in self.images]
        self.d_ids = torch.empty_like(ids)
        self.h_out = torch.empty((self.PAIRS, self.VOCAB), dtype=torch.float32).pin_memory()
        self.h2d_bytes = sum(t.numel() * 2 for t in self.h_images) + ids.numel() * 8
        self.d2h_bytes = self.h_out.numel() * 4
        self.T = T

    def step_device(self):
        self.out = self.model(input_ids=self.ids, attention_mask=None, images=self.images)

    def step_e2e(self):
        for d, h in zip(self.d_images, self.h_images):
            d.copy_(h, non_blocking=True)
        self.d_ids.copy_(self.h_ids, non_blocking=True)
        out = self.model(input_ids=self.d_ids, attention_mask=None, images=self.d_images)
        self.h_out.copy_(out.logits[:, -1, :], non_blocking=True)    # next-token distribution per pair

    def units_per_step(self):
        return self.PAIRS

    def dominant_kernel_ms(self, steps):
        """One extra instrumented step: CUDA events around every C-ABI launch, on the launch stream."""
        from visionllm_b200 import ops
        torch = self.torch
        torch.cuda.synchronize()
        ops.PROFILE = []
        self.step_device()
        torch.cuda.synchronize()
        prof, ops.PROFILE = ops.PROFILE, None
        agg, shapes = {}, {}
        for name, fl, by, e0, e1, *tag in prof:
            ms = e0.elapsed_time(e1)
            a = agg.setdefault(name, [0, 0.0, 0.0, 0.0])
            a[0] += 1; a[1] += ms; a[2] += fl; a[3] += by
            if name == "gemm" and tag and tag[0]:
                sh = shapes.setdefault(tag[0], [0, 0.0, fl])
                sh[0] += 1; sh[1] += ms
        self.breakdown = {k: {"launches": v[0], "ms": v[1], "tflops": v[2] / v[1] / 1e9 if v[1] else 0.0,
                              "gbps": v[3] / v[1] / 1e6 if v[1] else 0.0} for k, v in agg.items()}
        self.gemm_flops = agg["gemm"][2]
        self.gemm_ms = agg["gemm"][1]
        # the dominant kernel launch: the GEMM shape (M x N x K) with the largest total time in the step
        self.gemm_shapes = {k: {"launches": v[0], "ms_per_launch": v[1] / v[0], "tflops": v[2] / (v[1] / v[0]) / 1e9}
                            for k, v in sorted(shapes.items(), key=lambda kv: -kv[1][1])}
        self.top_shape = next(iter(self.gemm_shapes), None)
        return agg["gemm"][1]

    def roofline(self, kern_ms, peaks):
        pk = peaks["bf16_tflops_sustained"]
        top = self.gemm_shapes.get(self.top_shape) if self.top_shape else None
        if top is None:
            ach = self.gemm_flops / (kern_ms * 1e-3) / 1e12
            return {"kernel": "gemm_bf16_wgmma_kernel (all GEMM launches of one step, flop-weighted)", "bound": "tensor",
                    "achieved": ach, "peak": pk, "peak_source": peaks["source"], "unit": "TFLOP/s",
                    "frac": ach / pk, "traffic": None, "kernel_ms_per_step": kern_ms,
                    "algorithmic_flops_per_step": self.gemm_flops}
        # "MxNxK", or "b<n>xMxNxK" for a launch of n block-diagonal products (the attention-backward GEMMs of training)
        *nb, M, N, K = (int(v) for v in self.top_shape.lstrip("b").split("x"))
        nb = nb[0] if nb else 1
        all_ach = self.gemm_flops / (self.gemm_ms * 1e-3) / 1e12
        return {"kernel": f"gemm_bf16_wgmma_kernel at the step's dominant shape M x N x K = {self.top_shape} "
                          f"({top['launches']} launches per step)",
                "bound": "tensor", "achieved": top["tflops"], "peak": pk, "peak_source": peaks["source"],
                "unit": "TFLOP/s", "frac": top["tflops"] / pk,
                "algorithmic_flops_per_launch": top["tflops"] * 1e9 * top["ms_per_launch"], "ms_per_launch": top["ms_per_launch"],
                "traffic": None,                    # DRAM bytes of a launch: not measured
                "algorithmic_bytes_per_launch": 2.0 * nb * (M * K + N * K + M * N),
                "all_gemm_launches": {"achieved": all_ach, "frac": all_ach / pk, "kernel_ms_per_step": self.gemm_ms,
                                      "algorithmic_flops_per_step": self.gemm_flops},
                "top_shapes": dict(list(self.gemm_shapes.items())[:6])}

    def config(self):
        return {"workload": "BASELINE cfg 3: InternViT-6B(448, 5 anyres tiles of a 1024^2 image) + pixel-shuffle + "
                            "internvl_mlp + Vicuna-7B, T=1536 (1280 image + 256 text), fp32 logits all positions",
                "pairs_per_gpu_per_step": self.PAIRS, "seq_len": self.T, "tiles_per_image": 5,
                "l2_policy": "inputs_exceed_l2 (weights 25 GB, activations > 50 MB L2)",
                "parallelism": f"dp{self.world} (batch shard, no forward collective)",
                # stated, not hidden (VERDICT r1 weak #5): bf16 modules are held to the reference's OWN bf16 error, not to
                # the north-star's literal 1e-3 (one bf16 rounding is 2^-9); integer indices are exact
                "parity_rule": "bf16 modules: rel_l2(ours, ref_fp32) <= 1.5 x rel_l2(ref_bf16, ref_fp32) + 1e-3; "
                               "indices / integer outputs exact (tests/, DESIGN.md section 4)"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown}


class PairForward1TileWorkload(PairForwardWorkload):
    """SURVEY 8(d) cfg 3, the single-tile 'pad' variant: one 448^2 view per image (256 image tokens) + 256 text = T = 512."""
    TILES = 1

    def config(self):
        c = super().config()
        c.update(workload="BASELINE cfg 3, single-tile 'pad' variant: InternViT-6B(448, 1 tile) + pixel-shuffle + internvl_mlp + "
                          "Vicuna-7B, T=512 (256 image + 256 text), fp32 logits all positions", tiles_per_image=1)
        return c


class PairForwardClipWorkload(PairForwardWorkload):
    """SURVEY 8(d) cfg 3, the RELEASED 7B preset (vl/train/train.py:350-352, constant.py): CLIP-L/14-336 (24 layers, 1024
    wide, 577 tokens per tile, hidden_states[-2] without CLS) -> mlp2x_gelu bridge -> Vicuna-7B; 5 anyres tiles x 576 + 256
    text tokens = T = 3136."""
    TILE, TOK_PER_TILE = 336, 576
    BRIDGE, PIXEL_SHUFFLE, VIS_LAYER = "mlp2x_gelu", False, -2
    clip = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, image_size=336,
                patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)

    def vision_tower(self):
        from transformers import CLIPVisionConfig
        from visionllm_b200.clip import B200CLIPVisionModel
        return B200CLIPVisionModel(CLIPVisionConfig(**self.clip))

    def config(self):
        c = super().config()
        c.update(workload=f"BASELINE cfg 3, released-7B preset: CLIP-L/14-336 ({self.TILES} tile(s) of a 1024^2 image, "
                          f"hidden_states[-2]) + mlp2x_gelu + Vicuna-7B, T={self.T} ({self.TILES * 576} image + 256 text), "
                          "fp32 logits all positions", tiles_per_image=self.TILES)
        return c


class PairForwardClip1TileWorkload(PairForwardClipWorkload):
    """the released preset's single-tile 'pad' variant: T = 576 + 256 = 832."""
    TILES = 1


class GdinoHeadWorkload:
    """BASELINE cfg 4's region-decoder stage in isolation: Grounding-DINO-tiny enc/dec layers on the 4-level pyramid
    of a 1024^2 image (S = 21760), 80 class queries as text, 100 object queries: 6 x encoder layer (bi-attention
    fusion + text enhancer + MSDA deformable layer) + 6 x decoder layer (self-MHA, text cross-MHA, MSDA cross-attn,
    FFN).  Backbone / input projections are stubbed by synthetic features (they are cuDNN convs in the reference)."""
    metric = "gdino_encdec_images_per_sec_1024px"
    unit = "images/s"
    dtype = "bf16 (MSDA gather fp32)"
    N, Q, T = 8, 100, 80

    def __init__(self, rank, world, device):
        self.rank, self.world, self.device = rank, world, device

    def setup(self):
        import torch
        from types import SimpleNamespace
        from visionllm_b200.gdino import GroundingDinoDecoderLayer, GroundingDinoEncoderLayer
        self.torch = torch
        cfg = SimpleNamespace(d_model=256, encoder_attention_heads=8, decoder_attention_heads=8, encoder_ffn_dim=2048,
                              decoder_ffn_dim=2048, num_feature_levels=4, encoder_n_points=4, decoder_n_points=4,
                              dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, activation_function="relu")
        torch.manual_seed(0)
        dev = self.device
        self.enc = torch.nn.ModuleList([GroundingDinoEncoderLayer(cfg) for _ in range(6)]).to(dev, torch.bfloat16).eval()
        self.dec = torch.nn.ModuleList([GroundingDinoDecoderLayer(cfg) for _ in range(6)]).to(dev, torch.bfloat16).eval()
        g = torch.Generator(device=dev).manual_seed(7 + self.rank)
        shapes_l = GDINO_LEVELS_1024
        self.shapes = torch.tensor(shapes_l, dtype=torch.int64, device=dev)
        self.lsi = torch.cat((self.shapes.new_zeros(1), self.shapes.prod(1).cumsum(0)[:-1]))
        S = sum(h * w for h, w in shapes_l)
        N, Q, T = self.N, self.Q, self.T
        self.src = torch.randn(N, S, 256, device=dev, generator=g).bfloat16()
        self.pos = (torch.randn(N, S, 256, device=dev, generator=g) * 0.5).bfloat16()
        self.text = torch.randn(N, T, 256, device=dev, generator=g).bfloat16()
        refs = []
        for (H, W) in shapes_l:
            ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32),
                                    torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
            refs.append(torch.stack(((xs + 0.5) / W, (ys + 0.5) / H), -1).reshape(-1, 2))
        self.ref2 = torch.cat(refs, 0)[None, :, None, :].repeat(N, 1, 4, 1).contiguous()
        self.kpm = torch.zeros(N, S, dtype=torch.bool, device=dev)
        self.tmask = torch.zeros(N, T, dtype=torch.bool, device=dev)                 # no padded text
        self.tsa = torch.ones(N, T, T, dtype=torch.bool, device=dev)
        self.pids = torch.arange(T, device=dev)[None].repeat(N, 1)
        self.hs = torch.randn(N, Q, 256, device=dev, generator=g).bfloat16()
        self.qpos = (torch.randn(N, Q, 256, device=dev, generator=g) * 0.5).bfloat16()
        boxes = torch.rand(N, Q, 4, device=dev, generator=g) * 0.4 + 0.2
        self.ref4 = boxes[:, :, None, :].repeat(1, 1, 4, 1).contiguous()
        self.h_in = [t.cpu().pin_memory() for t in (self.src, self.pos, self.text)]
        self.d_in = [torch.empty_like(t) for t in (self.src, self.pos, self.text)]
        self.h_out = torch.empty((N, Q, 256), dtype=torch.bfloat16).pin_memory()
        self.h2d_bytes = sum(t.numel() * 2 for t in self.h_in)
        self.d2h_bytes = self.h_out.numel() * 2

    def _run(self, src, pos, text):
        v, t = src, text
        for layer in self.enc:
            (v, t), _ = layer(vision_features=v, vision_position_embedding=pos, spatial_shapes=self.shapes,
                              level_start_index=self.lsi, key_padding_mask=self.kpm, reference_points=self.ref2,
                              text_features=t, text_attention_mask=self.tmask, text_position_embedding=None,
                              text_self_attention_masks=self.tsa, text_position_ids=self.pids)
        h = self.hs
        for layer in self.dec:
            (h,) = layer(h, position_embeddings=self.qpos, reference_points=self.ref4, spatial_shapes=self.shapes,
                         level_start_index=self.lsi, vision_encoder_hidden_states=v,
                         vision_encoder_attention_mask=~self.kpm, text_encoder_hidden_states=t,
                         text_encoder_attention_mask=self.tmask)
        return h

    def step_device(self):
        self.out = self._run(self.src, self.pos, self.text)

    def step_e2e(self):
        for d, h in zip(self.d_in, self.h_in):
            d.copy_(h, non_blocking=True)
        self.h_out.copy_(self._run(*self.d_in), non_blocking=True)

    def units_per_step(self):
        return self.N

    def dominant_kernel_ms(self, steps):
        from visionllm_b200 import ops
        import visionllm_b200.msda as msda_mod
        torch = self.torch
        torch.cuda.synchronize()
        ops.PROFILE = []
        orig, orig16 = msda_mod.ms_deform_attn_forward, msda_mod.ms_deform_attn_forward_bf16
        msda_ms = []
        self.msda_value_bytes = 4

        def timed_msda(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r = orig(*a, **k); e1.record()
            msda_ms.append((e0, e1, a[0].shape, a[3].shape))
            return r

        def timed_msda16(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r = orig16(*a, **k); e1.record()
            msda_ms.append((e0, e1, a[0].shape, a[3].shape))
            self.msda_value_bytes = 2
            return r

        orig_fused = msda_mod.ms_deform_attn_forward_fused

        def timed_fused(*a, **k):                             # encoder modules: the fused module-input kernel
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r = orig_fused(*a, **k); e1.record()
            if r is not None:
                msda_ms.append((e0, e1, a[0].shape, (a[0].shape[0], a[0].shape[1])))
                self.msda_value_bytes = 2
                self.msda_fused = True
            return r

        import visionllm_b200.gdino as gd_mod
        gd_mod.msda_ext.ms_deform_attn_forward = timed_msda
        gd_mod.msda_ext.ms_deform_attn_forward_bf16 = timed_msda16
        gd_mod.msda_ext.ms_deform_attn_forward_fused = timed_fused
        try:
            self.step_device()
            torch.cuda.synchronize()
        finally:
            gd_mod.msda_ext.ms_deform_attn_forward = orig
            gd_mod.msda_ext.ms_deform_attn_forward_bf16 = orig16
            gd_mod.msda_ext.ms_deform_attn_forward_fused = orig_fused
        prof, ops.PROFILE = ops.PROFILE, None
        agg, shapes = {}, {}
        for name, fl, by, e0, e1, *tag in prof:
            ms = e0.elapsed_time(e1)
            a = agg.setdefault(name, [0, 0.0, 0.0, 0.0])
            a[0] += 1; a[1] += ms; a[2] += fl; a[3] += by
            if name == "gemm" and tag and tag[0]:
                sh = shapes.setdefault(tag[0], [0, 0.0, fl, by])
                sh[0] += 1; sh[1] += ms
        self.breakdown = {k: {"launches": v[0], "ms": v[1], "tflops": v[2] / v[1] / 1e9 if v[1] else 0.0,
                              "gbps": v[3] / v[1] / 1e6 if v[1] else 0.0} for k, v in agg.items()}
        self.gemm_shapes = {k: {"launches": v[0], "ms_total": v[1], "tflops": v[2] / (v[1] / v[0]) / 1e9,
                                "gbps": v[3] / (v[1] / v[0]) / 1e6}
                            for k, v in list(sorted(shapes.items(), key=lambda kv: -kv[1][1]))[:10]}
        enc_ms = [a.elapsed_time(b) for a, b, vs, ls in msda_ms if ls[1] == vs[1]]
        dec_ms = [a.elapsed_time(b) for a, b, vs, ls in msda_ms if ls[1] != vs[1]]
        self.breakdown["msda_encoder"] = {"launches": len(enc_ms), "ms": sum(enc_ms)}
        self.breakdown["msda_decoder"] = {"launches": len(dec_ms), "ms": sum(dec_ms)}
        self.msda_enc_ms = sum(enc_ms) / max(1, len(enc_ms))
        return self.msda_enc_ms if enc_ms else float("nan")

    def roofline(self, kern_ms, peaks):
        S = self.src.shape[1]
        vb = getattr(self, "msda_value_bytes", 4)            # bf16 value + bf16 out when the module takes the fast mode
        # value + (sampling_loc + attn_weight fp32 | fused: the bf16 offsets|logits projection row + reference points) + out
        side = (S * 8 * 16 * 3 * 2 + S * 4 * 2 * 4) if getattr(self, "msda_fused", False) else (S * 8 * 16 * 2 + S * 8 * 16) * 4
        alg = (S * 256 * vb + side + S * 256 * vb) * self.N
        ach = alg / (kern_ms * 1e-3) / 1e9
        kern = ("msda_fwd_win_kernel<bf16, bf16, 32, 16, 4, QP> (fused module input: softmax / offset normalisation / reference "
                "add inside the TMA-staged window gather; encoder launches inside the GDINO step)"
                if getattr(self, "msda_fused", False) else "msda_fwd_win/warp_kernel (encoder launches inside the GDINO step)")
        return {"kernel": kern, "bound": "hbm (nominal; issue-bound gather, DESIGN 6.2)",
                "achieved": ach, "peak": peaks["hbm_gbs"], "peak_source": peaks["source"], "unit": "GB/s",
                "frac": ach / peaks["hbm_gbs"], "traffic": None, "kernel_ms": kern_ms,
                "algorithmic_bytes_per_launch": alg}

    def config(self):
        return {"workload": "GDINO-tiny 6 enc + 6 dec layers, N=8 images, S=21760 (1024^2, 4 levels), 80 text "
                            "tokens, 100 queries (BASELINE cfg 4 region decoder, backbone/input_proj stubbed)",
                "l2_policy": "inputs_exceed_l2 (activations 8 x 21760 x 256 x ... > 50 MB L2)",
                "parallelism": f"dp{self.world}"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown, "top_gemm_shapes": getattr(self, "gemm_shapes", None)}


def build_gdino_stage(torch, device, hidden, backbone="b200"):
    """Grounding-DINO-tiny (Swin-T: embed 96, depths 2/2/6/2, window 7; 6 enc + 6 dec layers, d_model 256, FFN 2048,
    100 queries, mask head) as `visionllm_b200.gdino_model.B200GroundingDinoForObjectDetection`, random init."""
    from types import SimpleNamespace
    from transformers import SwinConfig
    from visionllm_b200.gdino_model import B200GroundingDinoForObjectDetection
    from visionllm_b200.swin import B200SwinBackbone
    bc = SwinConfig(image_size=224, embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=7,
                    out_features=["stage1", "stage2", "stage3", "stage4"])
    cfg = SimpleNamespace(backbone_config=bc, d_model=256, encoder_layers=6, decoder_layers=6, encoder_ffn_dim=2048,
                          decoder_ffn_dim=2048, encoder_attention_heads=8, decoder_attention_heads=8, num_queries=100,
                          num_feature_levels=4, encoder_n_points=4, decoder_n_points=4, dropout=0., attention_dropout=0.,
                          activation_dropout=0., activation_function="relu", mask_dim=256, norm="GN", l_hidden_size=hidden,
                          max_text_len=256, query_dim=4, two_stage=True, embedding_init_target=True,
                          two_stage_bbox_embed_share=False, decoder_bbox_embed_share=True, position_embedding_type="sine",
                          positional_embedding_temperature=20)
    torch.manual_seed(0)
    m = B200GroundingDinoForObjectDetection(cfg, backbone_model=B200SwinBackbone(bc) if backbone == "b200" else None)
    torch.nn.init.normal_(m.model.level_embed)
    return m.to(device, torch.bfloat16).eval()


class GdinoStageWorkload(GdinoHeadWorkload):
    """BASELINE cfg 4's WHOLE region-decoder stage on real inputs: 8 images [3,1024,1024] + text_query [8,80,4,4096]
    -> Swin-T backbone -> neck (GEMM + GroupNorm kernel) -> 6 encoder layers -> mask FPN -> two-stage top-k ->
    6 decoder layers -> class / box / mask heads -> detection post-processing (top-100 over Q x K)."""
    metric = "gdino_stage_images_per_sec_1024px"
    N_CLS = 80

    def setup(self):
        import torch
        self.torch = torch
        dev = self.device
        self.model = build_gdino_stage(torch, dev, 4096, backbone=os.environ.get("VLLM_BENCH_GDINO_BACKBONE", "b200"))
        g = torch.Generator(device=dev).manual_seed(7 + self.rank)
        N = self.N
        self.images = torch.randn(N, 3, 1024, 1024, device=dev, generator=g).bfloat16()
        self.tq = torch.randn(N, self.N_CLS, 4, 4096, device=dev, generator=g).bfloat16()
        self.tm = torch.ones(N, self.N_CLS, dtype=torch.bool, device=dev)
        self.h_in = [t.cpu().pin_memory() for t in (self.images, self.tq)]
        self.d_in = [torch.empty_like(t) for t in (self.images, self.tq)]
        self.h_out = torch.empty((N, 100, 6), dtype=torch.float32).pin_memory()
        self.h2d_bytes = sum(t.numel() * 2 for t in self.h_in)
        self.d2h_bytes = self.h_out.numel() * 4
        self.src = torch.empty(N, sum(h * w for h, w in GDINO_LEVELS_1024), 1, device="meta")     # shape only (roofline)
        self.graphed = None
        if os.environ.get("VLLM_BENCH_GRAPH", "1") != "0":
            from visionllm_b200.graphs import GraphedForward
            self.graphed = GraphedForward(lambda im, tq, tm: self.model(im, pixel_mask=None, text_query=tq, text_query_masks=tm))

    def _run(self, images, tq):
        from visionllm_b200 import gdino_heads as H, ops
        if self.graphed is not None and ops.PROFILE is None:          # CUDA-graph replay (eager for the profiling step)
            o = self.graphed(images, tq, self.tm)
        else:
            o = self.model(images, pixel_mask=None, text_query=tq, text_query_masks=self.tm)
        res, _, _ = H.post_process_det_gdino(o.logits, o.pred_boxes, [(1024, 1024)] * self.N, self.N_CLS, topk=100)
        self.masks = o.pred_masks
        return self.torch.stack([self.torch.cat([r["boxes"], r["scores"][:, None], r["labels"][:, None].float()], 1)
                                 for r in res])

    def step_device(self):
        self.out = self._run(self.images, self.tq)

    def config(self):
        return {"workload": "Grounding-DINO-tiny whole stage (BASELINE cfg 4 region decoder): N=8 images 1024^2, Swin-T "
                            "backbone on our kernels, neck, 6 enc + 6 dec layers (S=21760), 80 classes x 4 [EMB] text "
                            "queries, 100 object queries, box/class/mask heads, det post-processing",
                "l2_policy": "inputs_exceed_l2 (activations 8 x 65536 x 96 x ... > 50 MB L2)",
                "launch": "CUDA graph replay" if self.graphed is not None else "eager",
                "parallelism": f"dp{self.world}"}


class UniPoseStageWorkload(GdinoHeadWorkload):
    """SURVEY 8(f) rank 4 at the reference's real size: UniPose from pixels -- its own Swin-T backbone (`Joiner`, out indices
    1..3) -> input_proj (+ derived 4th level) -> 6 text-fused deformable encoder layers -> two-stage selection (900 queries)
    -> 2 box decoder layers -> top-50 -> 50 x (1 box + 68 keypoint) queries through 4 keypoint decoder layers -> box / class /
    keypoint heads; N images of 1024^2, [EMB] states of 1 object class + 17 keypoint classes (zero-padded to 100 slots each like
    mv2.py:803-809).  One CUDA graph when the capture succeeds (the forward has no host sync), eager otherwise."""
    metric = "unipose_stage_images_per_sec_1024px"
    N = 4

    def setup(self):
        import torch
        from visionllm_b200.unipose import B200UniPose
        from visionllm_b200.unipose_backbone import build_backbone
        self.torch = torch
        dev = self.device
        torch.manual_seed(0)
        bb = build_backbone("swin_T_224_1k", return_interm_indices=(1, 2, 3), hidden_dim=256)
        m = B200UniPose(hidden_dim=256, l_hidden_size=4096, backbone_channels=tuple(bb.num_channels), num_feature_levels=4,
                        num_queries=900, num_body_points=68, num_box_decoder_layers=2, nheads=8, backbone=bb,
                        num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=2048, dropout=0.0,
                        return_intermediate_dec=True, query_dim=4, deformable_encoder=True, deformable_decoder=True,
                        enc_n_points=4, dec_n_points=4, learnable_tgt_init=True, two_stage_type="standard", embed_init_tgt=True,
                        use_text_enhancer=True, use_fusion_layer=True, use_text_cross_attention=True, text_dropout=0.0,
                        fusion_dropout=0.0, fusion_droppath=0.0, decoder_sa_type="sa")
        self.model = m.to(dev, torch.bfloat16).eval()
        g = torch.Generator(device=dev).manual_seed(7 + self.rank)
        N = self.N
        self.images = torch.randn(N, 3, 1024, 1024, device=dev, generator=g).bfloat16()
        self.mask = torch.zeros(N, 1024, 1024, dtype=torch.bool, device=dev)
        obj = torch.zeros(N, 100, 4, 4096, device=dev, dtype=torch.bfloat16)
        kpt = torch.zeros(N, 100, 4, 4096, device=dev, dtype=torch.bfloat16)
        obj[:, :1] = torch.randn(N, 1, 4, 4096, device=dev, generator=g).bfloat16()
        kpt[:, :17] = torch.randn(N, 17, 4, 4096, device=dev, generator=g).bfloat16()
        om = torch.zeros(N, 100, dtype=torch.bool, device=dev); om[:, :1] = True
        km = torch.zeros(N, 100, dtype=torch.bool, device=dev); km[:, :17] = True
        self.tq = dict(obj_querys=obj, obj_query_masks=om, kpt_querys=kpt, kpt_query_masks=km)
        self.h_in = [t.cpu().pin_memory() for t in (self.images, obj, kpt)]
        self.d_in = [torch.empty_like(t) for t in (self.images, obj, kpt)]
        self.h_out = torch.empty((N, 50, 4 + 68 * 3), dtype=torch.float32).pin_memory()
        self.h2d_bytes = sum(t.numel() * 2 for t in self.h_in)
        self.d2h_bytes = self.h_out.numel() * 4
        self.graphed, self.launch = None, "eager"
        if os.environ.get("VLLM_BENCH_GRAPH", "1") != "0":
            # ~1800 launches per step, host-bound when eager: try one CUDA graph (the forward has no host sync); keep eager if
            # the capture is refused
            from visionllm_b200.graphs import GraphedForward
            gf = GraphedForward(lambda im, ob, kp: self._forward(im, ob, kp))
            try:
                gf(self.images, obj, kpt)
                torch.cuda.synchronize()
                self.graphed, self.launch = gf, "CUDA graph replay"
            except Exception as e:                                    # noqa: BLE001
                torch.cuda.synchronize()
                self.launch = f"eager (graph capture refused: {type(e).__name__}: {str(e)[:120]})"

    def _forward(self, images, obj, kpt):
        tq = dict(self.tq, obj_querys=obj, kpt_querys=kpt)
        o = self.model.forward_samples(images, self.mask, tq)
        return self.torch.cat((o.pred_boxes, o.pred_keypoints), -1)

    def _run(self, images, obj, kpt):
        from visionllm_b200 import ops
        if self.graphed is not None and ops.PROFILE is None:
            return self.graphed(images, obj, kpt)
        return self._forward(images, obj, kpt)

    def step_device(self):
        self.out = self._run(self.images, self.tq["obj_querys"], self.tq["kpt_querys"])

    def dominant_kernel_ms(self, steps):
        from visionllm_b200 import ops
        torch = self.torch
        torch.cuda.synchronize()
        ops.PROFILE = []
        self.step_device()
        torch.cuda.synchronize()
        prof, ops.PROFILE = ops.PROFILE, None
        agg = {}
        for name, fl, by, e0, e1, *tag in prof:
            a = agg.setdefault(name, [0, 0.0, 0.0, 0.0])
            a[0] += 1; a[1] += e0.elapsed_time(e1); a[2] += fl; a[3] += by
        self.breakdown = {k: {"launches": v[0], "ms": v[1], "tflops": v[2] / v[1] / 1e9 if v[1] else 0.0,
                              "gbps": v[3] / v[1] / 1e6 if v[1] else 0.0} for k, v in agg.items()}
        self.gemm_flops, self.gemm_ms = agg["gemm"][2], agg["gemm"][1]
        return self.gemm_ms

    def roofline(self, kern_ms, peaks):
        pk = peaks["bf16_tflops_sustained"]
        ach = self.gemm_flops / (kern_ms * 1e-3) / 1e12
        return {"kernel": "gemm_bf16_wgmma_kernel (all GEMM launches of one step, flop-weighted; short-K shapes, DESIGN 6.1)",
                "bound": "tensor", "achieved": ach, "peak": pk, "peak_source": peaks["source"], "unit": "TFLOP/s",
                "frac": ach / pk, "traffic": None, "kernel_ms_per_step": kern_ms, "algorithmic_flops_per_step": self.gemm_flops}

    def config(self):
        return {"workload": "UniPose whole stage from pixels (SURVEY 8f rank 4): N=4 images 1024^2, its Swin-T backbone, 6 enc + "
                            "6 dec layers (2 box + 4 keypoint), 900 -> 50 x 69 queries, 1 object class + 17 keypoint [EMB] classes",
                "l2_policy": "inputs_exceed_l2", "launch": self.launch, "parallelism": f"dp{self.world}"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown}


class PairForwardGdinoWorkload(PairForwardWorkload):
    """BASELINE cfg 4: cfg 3 + the Grounding-DINO region decoder head -- 80 classes x 4 [EMB] super-link tokens
    after a [DET] tool token each (T = 1280 image + 256 text + 80 x 5 = 1936), text_query gathered from the LLM's
    [EMB] hidden states, 100 object queries, 4-level features of the 1024^2 image, box / class / mask heads and
    the eval post-processing (top-k, //, %) inside the step."""
    metric = "img_text_pairs_per_sec_fwd_1024px_256tok_gdino100q"
    N_CLS = 80

    def setup(self):
        super().setup()
        torch = self.torch
        DET, EMB = 32003, 32010
        extra = torch.full((self.PAIRS, self.N_CLS * 5), EMB, dtype=self.ids.dtype, device=self.device)
        extra[:, 0::5] = DET
        self.ids = torch.cat([self.ids, extra], 1).contiguous()
        self.T = self.ids.shape[1]
        self.h_ids = self.ids.cpu().pin_memory()
        self.d_ids = torch.empty_like(self.ids)
        stage = build_gdino_stage(torch, self.device, 4096)
        if os.environ.get("VLLM_BENCH_GRAPH", "1") != "0":
            from visionllm_b200.graphs import GraphedForward
            graphed = GraphedForward(lambda pv, pm, tq, tm: stage(pv, pixel_mask=pm, text_query=tq, text_query_masks=tm))
            self.model.gdino = lambda pv, pixel_mask=None, text_query=None, text_query_masks=None, **kw: graphed(
                pv, pixel_mask, text_query, text_query_masks)
        else:
            self.model.gdino = stage
        self.model.use_gdino = True
        self.aug = torch.randn(self.PAIRS, 3, 1024, 1024, device=self.device).bfloat16()   # mmdet-normalised images_aug
        self.h_aug = self.aug.cpu().pin_memory()
        self.metas = [{"task": "det"} for _ in range(self.PAIRS)]        # the eval loop's img_metas (mv2.py:755-763)
        self.d_aug = torch.empty_like(self.aug)
        self.h2d_bytes = sum(t.numel() * 2 for t in self.h_images) + self.ids.numel() * 8 + self.aug.numel() * 2
        self.h_out = torch.empty((self.PAIRS, 100, 6), dtype=torch.float32).pin_memory()
        self.d2h_bytes = self.h_out.numel() * 4

    def _post(self, out):
        from visionllm_b200 import gdino_heads as H
        g = out.gdino_outputs
        res, idx, box_idx = H.post_process_det_gdino(g.logits, g.pred_boxes, [(1024, 1024)] * self.PAIRS, self.N_CLS,
                                                     topk=100)
        return self.torch.stack([self.torch.cat([r["boxes"], r["scores"][:, None], r["labels"][:, None].float()], 1)
                                 for r in res])

    def step_device(self):
        self.out = self._post(self.model(input_ids=self.ids, attention_mask=None, images=self.images, images_aug=self.aug,
                                         img_metas=self.metas))

    def step_e2e(self):
        for d, h in zip(self.d_images, self.h_images):
            d.copy_(h, non_blocking=True)
        self.d_ids.copy_(self.h_ids, non_blocking=True)
        self.d_aug.copy_(self.h_aug, non_blocking=True)
        out = self._post(self.model(input_ids=self.d_ids, attention_mask=None, images=self.d_images, images_aug=self.d_aug,
                                    img_metas=self.metas))
        self.h_out.copy_(out, non_blocking=True)                     # boxes, scores, labels of the top-100 detections

    def config(self):
        c = super().config()
        c["workload"] = ("BASELINE cfg 4: cfg 3 + GDINO region decoder (80 classes x ([DET] + 4 [EMB]), 100 queries, "
                         "Swin-T backbone + neck + 6 enc + 6 dec layers on the 1024^2 images_aug), heads + det post-processing in the step")
        c["seq_len"] = self.T
        return c


class LlmTpWorkload(PairForwardWorkload):
    """BASELINE cfg 5 (forward): Vicuna-7B split over the GPUs of the box (visionllm_b200/tp.py: tensor-parallel
    attention + sequence-parallel MLP, one reduce-scatter + one all-gather per layer fused into the o_proj GEMM
    epilogue and the RMSNorm kernel, no NCCL on the data path), 8 sequences of 2048 mixed visual/text tokens per step
    for the WHOLE job (strong scaling: the same 16384 tokens at any world size), fp32 logits for every position."""
    metric = "llm_tp_fwd_tokens_per_sec_2048tok"
    unit = "tokens/s"
    dtype = "bf16"
    SEQS, T = 8, 2048
    MICRO = 2              # micro-batches on their own streams / exchange buffers (tp.forward_pipelined); 1 = plain forward

    def setup(self):
        import torch
        import torch.distributed as dist
        from transformers import LlamaConfig
        from visionllm_b200 import tp
        self.torch = torch
        cfg = LlamaConfig(**self.llm)
        M = self.SEQS * self.T
        if self.world > 1:
            self.comm = tp.PeerComm.from_process_group(M, cfg.hidden_size, self.device)
        else:
            self.comm = tp.PeerComm.virtual(1, M, cfg.hidden_size, self.device)[0]
        self.model = tp.TPLlamaForCausalLM.random_init(cfg, self.comm, self.device, seed=0)
        self.micro = None
        if self.MICRO > 1 and self.world > 1:
            mk = (lambda: tp.PeerComm.from_process_group(M // self.MICRO, cfg.hidden_size, self.device))
            self.micro = [mk() for _ in range(self.MICRO)]
        g = torch.Generator(device=self.device).manual_seed(1234)           # the same batch on every rank (TP)
        self.ids = torch.randint(0, 32000, (self.SEQS, self.T), device=self.device, generator=g)
        self.emb = torch.nn.functional.embedding(self.ids, self.model.shards["embed"])
        self.h_ids = self.ids.cpu().pin_memory()
        self.d_ids = torch.empty_like(self.ids)
        self.h_out = torch.empty((self.SEQS, cfg.hidden_size), dtype=torch.bfloat16).pin_memory()
        self.h2d_bytes = self.ids.numel() * 8
        self.d2h_bytes = self.h_out.numel() * 2
        self.dist = dist if self.world > 1 else None

    def step_device(self):
        if self.micro:
            self.out = self.model.forward_pipelined(self.micro, inputs_embeds=self.emb)
        else:
            self.out = self.model(inputs_embeds=self.emb)

    def step_e2e(self):
        self.d_ids.copy_(self.h_ids, non_blocking=True)
        if self.micro:
            out = self.model.forward_pipelined(self.micro, input_ids=self.d_ids)
        else:
            out = self.model(input_ids=self.d_ids)
        self.h_out.copy_(out.last_hidden_state[:, -1, :], non_blocking=True)

    def units_per_step(self):
        return self.SEQS * self.T / self.world        # bench.py multiplies by world: the job's tokens per step

    def config(self):
        return {"workload": "BASELINE cfg 5 forward: Vicuna-7B, 8 x 2048-token sequences per step for the whole job, "
                            "tensor-parallel attention + sequence-parallel MLP over peer memory, fp32 logits all positions",
                "global_batch": self.SEQS, "seq_len": self.T,
                "l2_policy": "inputs_exceed_l2 (weights 13.5 GB / TP shard + replicated MLP, activations > 50 MB L2)",
                "parallelism": f"tp{self.world} (heads) x sp{self.world} (token rows); 1 reduce-scatter + 1 all-gather "
                               "per layer inside the GEMM epilogue / norm kernel",
                "micro_batches": self.MICRO if self.micro else 1}

    def extra(self):
        return {"kernel_breakdown": self.breakdown, "scaling": "strong"}


class LlmTpPlainWorkload(LlmTpWorkload):
    """llm_tp without micro-batch pipelining (the r1 schedule), for the comparison."""
    MICRO = 1


class InternImageHWorkload(PairForwardWorkload):
    """The alternative GDINO backbone of BASELINE cfg 4 (SURVEY 8a-a13): InternImage-H (gd.py:5154-5170: 320 channels,
    depths [6, 6, 32, 6], groups [10, 20, 40, 80], 5x5 depthwise branch, DCNv3 core, centre-feature scale), random init,
    bf16, 4 images of 1024^2 per GPU per step through `visionllm_b200.internimage.build_internimage_h`, all four level
    maps returned."""
    metric = "internimage_h_backbone_images_per_sec_1024px"
    unit = "images/s"
    dtype = "bf16 (DCNv3 core fp32)"
    IMAGES = 4

    def setup(self):
        import torch
        from visionllm_b200.internimage import build_internimage_h
        self.torch = torch
        with torch.device("meta"):
            m = build_internimage_h()
        m = m.to_empty(device=self.device).to(torch.bfloat16)
        g = torch.Generator(device=self.device).manual_seed(0)
        with torch.no_grad():
            for name, p in m.named_parameters():
                last = name.split(".")[-1]
                if p.dim() <= 1:
                    p.fill_(1.0) if (last == "weight") else p.zero_()
                else:
                    fan_in = p[0].numel()
                    p.copy_(torch.randn(p.shape, device=self.device, generator=g, dtype=torch.float32) / fan_in ** 0.5)
        self.model = m.eval()
        gi = torch.Generator(device=self.device).manual_seed(1234 + self.rank)
        self.images = torch.randn(self.IMAGES, 3, 1024, 1024, device=self.device, generator=gi).bfloat16()
        self.h_images = self.images.cpu().pin_memory()
        self.d_images = torch.empty_like(self.images)
        self.h_out = torch.empty((self.IMAGES, 32, 32, 2560), dtype=torch.bfloat16).pin_memory()
        self.h2d_bytes = self.images.numel() * 2
        self.d2h_bytes = self.h_out.numel() * 2
        from visionllm_b200.graphs import GraphedForward
        self.fwd = GraphedForward(lambda x: tuple(self.model(x)))     # ~2500 launches per step: replay, not Python
        self.eager = False

    def step_device(self):
        self.out = self.model(self.images) if self.eager else self.fwd(self.images)

    def step_e2e(self):
        self.d_images.copy_(self.h_images, non_blocking=True)
        out = self.fwd(self.d_images)
        self.h_out.copy_(out[-1], non_blocking=True)

    def units_per_step(self):
        return self.IMAGES

    def dominant_kernel_ms(self, steps):
        self.eager = True                       # per-launch CUDA events need the eager launches
        try:
            return super().dominant_kernel_ms(steps)
        finally:
            self.eager = False

    def config(self):
        return {"workload": "InternImage-H backbone forward (GDINO backbone option of BASELINE cfg 4): 4 x 1024^2 images, "
                            "strides 4/8/16/32 maps of 320/640/1280/2560 channels",
                "images_per_gpu_per_step": self.IMAGES, "launch": "CUDA graph replay",
                "l2_policy": "inputs_exceed_l2 (weights 2.2 GB, level-0 activations 168 MB per tensor > 50 MB L2)",
                "parallelism": f"dp{self.world} (batch shard, no forward collective)"}


class LlmTrainWorkload(PairForwardWorkload):
    """BASELINE cfg 5's "fwd+bwd step" on the training-side path (visionllm_b200/train.py): Vicuna-7B random-init bf16,
    SEQS x 2048 mixed visual/text tokens per GPU per step (the first 1536 positions visual: no language loss), loss = CE on
    the text positions (modeling_visionllmv2.py:741-757), forward + backward of every decoder op on this repo's kernels
    (wgmma GEMMs incl. MN-major dgrad / wgrad and the batched attention backward; row backward kernels; fused CE).  No
    optimizer step (stated).  N GPUs: data-parallel replicas with ONE bf16 gradient all-reduce (NCCL) per step inside the
    timed region -- the tensor-parallel exchange of tp.py is forward-only."""
    metric = "llm_train_fwd_bwd_tokens_per_sec_2048tok"
    unit = "tokens/s"
    dtype = "bf16 (fp32 accumulate, fp32 logits / loss)"
    SEQS, T = 4, 2048

    def setup(self):
        import torch
        import torch.distributed as dist
        from transformers import LlamaConfig
        from visionllm_b200.llama import B200LlamaForCausalLM
        from visionllm_b200.train import B200LlamaForCausalLMTrain
        self.torch = torch
        cfg = LlamaConfig(**self.llm)
        with torch.device("meta"):
            lm = B200LlamaForCausalLM(cfg)
        lm = lm.to_empty(device=self.device).to(torch.bfloat16)
        g = torch.Generator(device=self.device).manual_seed(0)
        with torch.no_grad():
            for name, p in lm.named_parameters():
                if "norm" in name:
                    p.fill_(1.0)
                else:
                    p.copy_(torch.randn(p.shape, device=self.device, generator=g, dtype=torch.float32) * 0.02)
        self.lm = lm
        self.model = B200LlamaForCausalLMTrain(lm)
        gi = torch.Generator(device=self.device).manual_seed(1234 + self.rank)
        self.ids = torch.randint(0, 32000, (self.SEQS, self.T), device=self.device, generator=gi)
        self.labels = self.ids.clone()
        self.labels[:, :1536] = -100
        self.h_ids = self.ids.cpu().pin_memory()
        self.h_labels = self.labels.cpu().pin_memory()
        self.d_ids, self.d_labels = torch.empty_like(self.ids), torch.empty_like(self.labels)
        self.h_out = torch.empty((1,), dtype=torch.float32).pin_memory()
        self.h2d_bytes = self.ids.numel() * 16
        self.d2h_bytes = 4
        self.dist = dist if self.world > 1 else None
        self.params = [p for n, p in lm.named_parameters() if n != "model.embed_tokens.weight"]

    def _step(self, ids, labels):
        torch = self.torch
        for p in self.params:
            p.grad = None
        with torch.no_grad():
            emb = torch.nn.functional.embedding(ids, self.lm.model.embed_tokens.weight)
        loss, _, _ = self.model(emb.requires_grad_(True), labels)
        loss.backward()
        if self.dist is not None:                                  # the exchange step of data-parallel training
            flat = torch.cat([p.grad.reshape(-1) for p in self.params])
            self.dist.all_reduce(flat)
        return loss.detach()

    def step_device(self):
        self.out = self._step(self.ids, self.labels)

    def step_e2e(self):
        self.d_ids.copy_(self.h_ids, non_blocking=True)
        self.d_labels.copy_(self.h_labels, non_blocking=True)
        self.h_out.copy_(self._step(self.d_ids, self.d_labels).reshape(1), non_blocking=True)

    def units_per_step(self):
        return self.SEQS * self.T

    def config(self):
        return {"workload": f"BASELINE cfg 5 fwd+bwd (training-side path): Vicuna-7B, {self.SEQS} x 2048-token sequences per GPU "
                            "per step, CE loss on the 512 text positions, forward + backward on this repo's kernels, no optimizer",
                "global_batch": self.SEQS * self.world, "seq_len": self.T,
                "l2_policy": "inputs_exceed_l2 (weights 13.5 GB + saved activations ~40 GB)",
                "parallelism": f"dp{self.world} (one bf16 gradient all-reduce per step)" if self.world > 1 else "dp1"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown}


class LlmTpTrainWorkload(LlmTrainWorkload):
    """BASELINE cfg 5 as written: Vicuna-7B tensor-parallel over the GPUs of the box, fwd+bwd (visionllm_b200/tp_train.py:
    Megatron split, two NCCL all-reduces per layer forward + two backward over NVLink, every compute op a kernel of this
    repo), 4 x 2048-token sequences per step for the WHOLE job at any world size (strong scaling).  Four sequences, not
    the eight of the forward-only llm_tp: the saved activations of 16384 tokens and the unsharded weights and gradients do
    not fit the 80 GB of one H100 at world size 1 (out of memory there), 8192 tokens do (llm_train: 55.5 GB peak)."""
    metric = "llm_tp_train_fwd_bwd_tokens_per_sec_2048tok"
    SEQS = 4

    def setup(self):
        import torch
        import torch.distributed as dist
        from transformers import LlamaConfig
        from visionllm_b200 import tp_train
        self.torch = torch
        cfg = LlamaConfig(**self.llm)
        g = torch.Generator(device=self.device).manual_seed(0)           # the same full weights on every rank, then sharded
        H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
        r = lambda *sh: (torch.randn(*sh, device=self.device, generator=g, dtype=torch.float32) * 0.02).to(torch.bfloat16)  # noqa: E731
        sd = {"model.norm.weight": torch.ones(H, device=self.device, dtype=torch.bfloat16), "lm_head.weight": r(V, H)}
        self.embed = r(V, H)
        for i in range(cfg.num_hidden_layers):
            p = f"model.layers.{i}."
            sd.update({p + "self_attn.q_proj.weight": r(H, H), p + "self_attn.k_proj.weight": r(H, H),
                       p + "self_attn.v_proj.weight": r(H, H), p + "self_attn.o_proj.weight": r(H, H),
                       p + "mlp.gate_proj.weight": r(I, H), p + "mlp.up_proj.weight": r(I, H), p + "mlp.down_proj.weight": r(H, I),
                       p + "input_layernorm.weight": torch.ones(H, device=self.device, dtype=torch.bfloat16),
                       p + "post_attention_layernorm.weight": torch.ones(H, device=self.device, dtype=torch.bfloat16)})
            if self.world > 1:                                           # keep only this rank's shard of the layer alive
                pass
        shards = tp_train.shard_for_training(sd, cfg, self.rank if self.world > 1 else 0, self.world)
        del sd
        torch.cuda.empty_cache()
        self.model = tp_train.TPLlamaTrain(cfg, shards, group=None)
        self.params = list(shards.parameters())
        gi = torch.Generator(device=self.device).manual_seed(1234)       # the same batch on every rank (TP)
        self.ids = torch.randint(0, 32000, (self.SEQS, self.T), device=self.device, generator=gi)
        self.labels = self.ids.clone()
        self.labels[:, :1536] = -100
        self.h_ids, self.h_labels = self.ids.cpu().pin_memory(), self.labels.cpu().pin_memory()
        self.d_ids, self.d_labels = torch.empty_like(self.ids), torch.empty_like(self.labels)
        self.h_out = torch.empty((1,), dtype=torch.float32).pin_memory()
        self.h2d_bytes = self.ids.numel() * 16
        self.d2h_bytes = 4
        self.dist = dist if self.world > 1 else None

    def _step(self, ids, labels):
        torch = self.torch
        for p in self.params:
            p.grad = None
        with torch.no_grad():
            emb = torch.nn.functional.embedding(ids, self.embed)
        loss, _, _ = self.model(emb.requires_grad_(True), labels)
        loss.backward()
        return loss.detach()

    def units_per_step(self):
        return self.SEQS * self.T / self.world        # bench.py multiplies by world: the job's tokens per step

    def config(self):
        return {"workload": "BASELINE cfg 5: Vicuna-7B tensor-parallel fwd+bwd, 4 x 2048-token sequences per step for the whole "
                            "job, CE loss on the 512 text positions of each, no optimizer",
                "global_batch": self.SEQS, "seq_len": self.T,
                "l2_policy": "inputs_exceed_l2",
                "parallelism": f"tp{self.world}: column / row parallel attention + MLP, 2 NCCL all-reduces per layer forward and "
                               "2 backward (north_star: 'a single NCCL allreduce over NVLink per layer' per block)"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown, "scaling": "strong"}


class Cfg1Workload:
    """BASELINE cfg 1 ("single 224x224 image + 16-token prompt, ViT-B + 1-layer LLM stub, CPU reference fwd"): ViT-B-size
    InternViT -> mlp2x_gelu -> 1-layer Llama -> [EMB] gather -> whole Grounding-DINO stage (Swin backbone, 6 + 6 layers,
    100 queries, S = 1045) through `B200VisionLLMv2Model.forward` -- the configuration whose reference CPU forward is
    runnable, so the CPU baseline beside it is MEASURED on the same workload, not extrapolated
    (tests/golden/cfg1_common.py holds the shapes; parity: tests/test_cfg1_e2e_gpu.py, tests/test_cfg1_logic_cpu.py)."""
    metric = "img_text_pairs_per_sec_fwd_cfg1_224px_16tok"
    unit = "pairs/s"
    dtype = "bf16"

    def __init__(self, rank, world, device):
        self.rank, self.world, self.device = rank, world, device

    @staticmethod
    def _common():
        import sys
        g = os.path.join(ROOT, "tests", "golden")
        if g not in sys.path:
            sys.path.insert(0, g)
        import cfg1_common
        return cfg1_common

    def setup(self):
        import torch
        self.torch = torch
        C = self._common()
        self.model = C.build_b200_model(None, device=self.device, dtype=torch.bfloat16)
        ids, image, aug = C.inputs()
        self.h = [ids.pin_memory(), image.bfloat16().pin_memory(), aug[0].bfloat16().pin_memory()]
        self.d = [t.to(self.device) for t in self.h]
        self.mask = torch.ones_like(self.d[0])
        self.metas = [{"task": "det"}]
        self.h_out = torch.empty((1, 100, 6), dtype=torch.float32).pin_memory()
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in self.h)
        self.d2h_bytes = self.h_out.numel() * 4
        self.n_cls = C.N_CLS

    def _run(self, ids, image, aug):
        from visionllm_b200 import gdino_heads as H
        out = self.model(input_ids=ids, attention_mask=self.mask, images=image, images_aug=[aug], img_metas=self.metas)
        g = out.gdino_outputs
        res, _, _ = H.post_process_det_gdino(g.logits, g.pred_boxes, [(224, 224)], self.n_cls, topk=100)
        r = res[0]
        return self.torch.cat([r["boxes"], r["scores"][:, None], r["labels"][:, None].float()], 1)[None]

    def step_device(self):
        self.out = self._run(*self.d)

    def step_e2e(self):
        for d, h in zip(self.d, self.h):
            d.copy_(h, non_blocking=True)
        self.h_out.copy_(self._run(*self.d), non_blocking=True)

    def units_per_step(self):
        return 1

    dominant_kernel_ms = PairForwardWorkload.dominant_kernel_ms

    def roofline(self, kern_ms, peaks):
        r = PairForwardWorkload.roofline(self, kern_ms, peaks)
        r["note"] = "toy widths (768 / 512 / 256): launch-latency bound, the GEMM fraction is not the story of this config"
        return r

    def config(self):
        return {"workload": "BASELINE cfg 1: 1 x (224^2 image, 256 <im_patch> + 16 text + 5 x ([DET] + 4 [EMB]) tokens), "
                            "ViT-B-size InternViT (768/12 layers) + mlp2x_gelu + 1-layer Llama (512) + GDINO (Swin embed 48, "
                            "6 + 6 layers, 100 queries, S = 1045) + det post-processing",
                "l2_policy": "fits_in_l2 (the whole model is ~60 MB: stated, this config exists for parity and the CPU timing)",
                "parallelism": f"dp{self.world}"}

    def extra(self):
        return {"kernel_breakdown": self.breakdown}


# --------------------------------------------------------------------------------------
# Extra objects of the DEFAULT bench line (VERDICT r1 1c): the other half of BASELINE.json's metric ("deform-attn HBM
# GB/s", cfg 2b) and, under torchrun, cfg 5 (LLM tensor parallelism) -- so that the driver's BENCH / SCALE records carry
# them.  Both run AFTER the timed regions of the main workload.
# --------------------------------------------------------------------------------------
def _event_ms(torch, fn, reps, warm=3, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps


def msda_extra(device, reps=20):
    """MSDA forward at the cfg-2b encoder shape on THIS GPU: our kernel (fp32 reference layout = the parity path, and
    bf16 value = the GDINO modules' path) and, when oracle/_ref/msda holds it, the reference's own CUDA kernel
    recompiled for sm_90.  CUDA events per launch, L2 flushed between launches; GB/s on the algorithmic bytes
    (SURVEY 8d: value + sampling_loc + attn_weight once, output once)."""
    import torch
    import visionllm_b200.msda as ext
    peaks = measured_peaks()
    N = 8
    value, shapes, lsi, loc, attw = msda_encoder_inputs(torch, N, device, 1234)
    hs = shapes.cpu()
    S = value.shape[1]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    alg32 = (value[0].numel() + loc[0].numel() + attw[0].numel() + S * 256) * 4 * N
    alg16 = (value[0].numel() * 2 + loc[0].numel() * 4 + attw[0].numel() * 4 + S * 256 * 2) * N

    def row(ms, alg, kernel, traffic):
        return {"kernel": kernel, "ms": ms, "GBps": alg / ms / 1e6, "frac": alg / ms / 1e6 / peaks["hbm_gbs"],
                "algorithmic_bytes_per_launch": alg, "traffic": traffic}

    out = {"workload": "msda_fwd encoder shape (BASELINE cfg 2b): N=8 S=Lq=21760 M=8 D=32 L=4 P=4, L2 flushed between launches",
           "bound": "hbm (nominal; the gather is L1/shared-memory wavefront bound, DESIGN 6.2)", "peak": peaks["hbm_gbs"],
           "peak_source": peaks["source"], "unit": "GB/s"}
    ms = _event_ms(torch, lambda: ext.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64, host_shapes=hs), reps,
                   flush=flush)
    out["fp32"] = row(ms, alg32, "msda_fwd_warp_kernel<8, 16, 16, 16, 4, float, float> (global-memory patch kernel: the default for "
                                 "fp32 rows; the TMA-staged window kernel is variant 33)",
                      None)
    v16 = value.bfloat16()
    ms = _event_ms(torch, lambda: ext.ms_deform_attn_forward_bf16(v16, shapes, lsi, loc, attw), reps, flush=flush)
    out["bf16_value"] = row(ms, alg16, "msda_fwd_win_kernel<__nv_bfloat16, __nv_bfloat16, 32, 16, 4> (TMA-staged windows, 16 x 32 patch)",
                            None)
    try:
        import importlib.util
        path = os.path.join(ROOT, "oracle", "_ref", "msda", "MultiScaleDeformableAttention.so")
        if os.path.exists(path):
            spec = importlib.util.spec_from_file_location("MultiScaleDeformableAttention", path)
            ref = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(ref)
            ms = _event_ms(torch, lambda: ref.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64), 5, warm=2,
                           flush=flush)
            r = row(ms, alg32, "ms_deformable_im2col_gpu_kernel (reference unipose/ops CUDA source recompiled for sm_90)", None)
            mine = ext.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64, host_shapes=hs)
            theirs = ref.ms_deform_attn_forward(value, shapes, lsi, loc, attw, 64)
            r["max_abs_diff_ours_vs_reference_kernel"] = float((mine - theirs).abs().max())
            out["reference_cuda_kernel_fp32"] = r
        else:
            out["reference_cuda_kernel_fp32"] = {"unavailable": "oracle/_ref/msda not built (python oracle/build_msda_ref.py)"}
    except Exception as e:                                # the reference arm is evidence, never a dependency
        out["reference_cuda_kernel_fp32"] = {"unavailable": f"{type(e).__name__}: {e}"[:200]}
    return out


def tp_parity_check(rank, world, device):
    """world-process parity of the tensor-parallel LLM over real IPC peer memory: a 3-layer Llama (hidden 1024, 8 heads
    x 128) sharded over the ranks vs the unsharded B200 Llama on the same weights / inputs; max rel_l2 over ranks."""
    import torch
    import torch.distributed as dist
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200 import tp
    from visionllm_b200.llama import B200LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2752, num_hidden_layers=3, num_attention_heads=8,
                      num_key_value_heads=8, vocab_size=1024, rms_norm_eps=1e-5, max_position_embeddings=1024)
    torch.manual_seed(0)
    sd = {k: v.to(torch.bfloat16).float() for k, v in LlamaForCausalLM(cfg).state_dict().items()}
    B, T, H = 2, 512, 1024
    emb = (torch.randn(B, T, H, generator=torch.Generator().manual_seed(1)) * 0.5).bfloat16().to(device)
    single = B200LlamaForCausalLM(cfg)
    single.load_state_dict(sd)
    single = single.to(device, torch.bfloat16).eval()
    one = single(inputs_embeds=emb, output_hidden_states=True)
    comm = tp.PeerComm.from_process_group(B * T, H, device)
    m = tp.TPLlamaForCausalLM.from_full_state_dict(cfg, comm, sd, device=device)
    rel = lambda a, b: float(torch.linalg.norm(a.float() - b.float()) / torch.linalg.norm(b.float()))  # noqa: E731
    e1 = e2 = 0.0
    for _ in range(3):                                    # repeated forwards: buffer reuse / epoch counters
        out = m(inputs_embeds=emb)
        torch.cuda.synchronize()
        lo, hi = out.row_range
        e1 = max(e1, rel(out.last_hidden_state, one.hidden_states[-1]))
        e2 = max(e2, rel(out.logits_local, one.logits.reshape(B * T, -1)[lo:hi]))
    t = torch.tensor([e1, e2], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    del m, comm, single
    return {"what": f"{world}-process TP forward (3-layer Llama 1024/8x128, 2 x 512 tokens, 3 repeated forwards over IPC "
                    "peer memory) vs the unsharded B200 Llama, max over ranks",
            "rel_l2_last_hidden": float(t[0]), "rel_l2_logits": float(t[1]), "tolerance": 1e-2,
            "ok": bool(t[0] < 1e-2 and t[1] < 1e-2)}


def tp_extra(rank, world, device, steps=10, warmup=3):
    """BASELINE cfg 5 (forward) under the SAME torchrun launch as the default line: parity check, then the llm_tp
    workload (strong scaling: 8 x 2048 tokens per step for the whole job), CUDA events, max over ranks."""
    import torch
    import torch.distributed as dist
    res = {"parity": tp_parity_check(rank, world, device)}
    wl = LlmTpWorkload(rank=rank, world=world, device=device)
    wl.setup()
    for _ in range(warmup):
        wl.step_device()
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        wl.step_device()
    e1.record()
    dist.barrier(); torch.cuda.synchronize()
    ms = max_over_ranks(e0.elapsed_time(e1), dist, "cuda") / steps
    tokens = wl.SEQS * wl.T
    flops = tokens * (32 * 2 * (4 * 4096 * 4096 + 3 * 4096 * 11008) + 2 * 4096 * wl.VOCAB) + 32 * 4 * wl.SEQS * wl.T * wl.T * 4096 * 0.5
    peaks = measured_peaks()
    res.update({"metric": wl.metric, "value": tokens / (ms * 1e-3), "unit": wl.unit, "ms_per_step": ms, "steps": steps,
                "warmup": warmup, "scaling": "strong", "config": wl.config(),
                "tflops_per_gpu": flops / world / (ms * 1e-3) / 1e12,
                "frac_of_sustained_bf16_peak": flops / world / (ms * 1e-3) / 1e12 / peaks["bf16_tflops_sustained"]})
    del wl
    torch.cuda.empty_cache()
    try:                                                    # the r1 schedule (no micro-batch pipelining) beside it
        wp = LlmTpPlainWorkload(rank=rank, world=world, device=device)
        wp.setup()
        for _ in range(warmup):
            wp.step_device()
        dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            wp.step_device()
        e1.record()
        dist.barrier(); torch.cuda.synchronize()
        res["plain_schedule_ms_per_step"] = max_over_ranks(e0.elapsed_time(e1), dist, "cuda") / steps
        del wp
    except Exception as e:
        res["plain_schedule_ms_per_step"] = f"{type(e).__name__}: {e}"[:200]
    torch.cuda.empty_cache()
    try:
        res["train"] = tp_train_extra(rank, world, device)
    except Exception as e:                                  # evidence, never a dependency of the line
        res["train"] = {"error": f"{type(e).__name__}: {e}"[:300]}
    torch.cuda.empty_cache()
    return res


def tp_train_extra(rank, world, device, steps=5, warmup=2):
    """cfg 5 fwd+bwd under the same launch: (1) parity of the tensor-parallel loss / input gradient against the unsharded
    training path on a 3-layer model, (2) the llm_tp_train workload (Vicuna-7B, 4 x 2048 tokens per step for the job)."""
    import torch
    import torch.distributed as dist
    from transformers import LlamaConfig, LlamaForCausalLM
    from visionllm_b200 import tp_train
    from visionllm_b200.llama import B200LlamaForCausalLM
    from visionllm_b200.train import B200LlamaForCausalLMTrain
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2816, num_hidden_layers=3, num_attention_heads=8,
                      num_key_value_heads=8, vocab_size=1024, rms_norm_eps=1e-5, max_position_embeddings=1024)
    torch.manual_seed(0)
    sd = {k: v.to(torch.bfloat16) for k, v in LlamaForCausalLM(cfg).state_dict().items()}
    B, T = 2, 512
    gen = torch.Generator().manual_seed(1)
    emb = (torch.randn(B, T, 1024, generator=gen) * 0.5).bfloat16().to(device)
    labels = torch.randint(0, 1024, (B, T), generator=gen).to(device)
    labels[:, :200] = -100
    single = B200LlamaForCausalLM(cfg)
    single.load_state_dict({k: v.float() for k, v in sd.items()})
    single = single.to(device, torch.bfloat16)
    e1 = emb.clone().requires_grad_(True)
    l1, _, _ = B200LlamaForCausalLMTrain(single)(e1, labels)
    l1.backward()
    shards = tp_train.shard_for_training({k: v.to(device) for k, v in sd.items()}, cfg, rank, world)
    e2 = emb.clone().requires_grad_(True)
    l2, _, _ = tp_train.TPLlamaTrain(cfg, shards)(e2, labels)
    l2.backward()
    rel = lambda a, b: float(torch.linalg.norm(a.float() - b.float()) / torch.linalg.norm(b.float()))  # noqa: E731
    t = torch.tensor([abs(float(l2) - float(l1)) / abs(float(l1)), rel(e2.grad, e1.grad)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    res = {"parity": {"what": f"{world}-way tensor-parallel fwd+bwd (3-layer Llama 1024/8x128, 2 x 512 tokens) vs the unsharded "
                              "training path on the same weights: relative loss difference, rel_l2 of d loss / d inputs_embeds; "
                              "max over ranks",
                      "loss_rel_diff": float(t[0]), "dinputs_rel_l2": float(t[1]), "ok": bool(t[0] < 5e-3 and t[1] < 3e-2)}}
    del single, shards
    torch.cuda.empty_cache()
    wl = LlmTpTrainWorkload(rank=rank, world=world, device=device)
    wl.setup()
    for _ in range(warmup):
        wl.step_device()
    dist.barrier(); torch.cuda.synchronize()
    e0, e1_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        wl.step_device()
    e1_.record()
    dist.barrier(); torch.cuda.synchronize()
    ms = max_over_ranks(e0.elapsed_time(e1_), dist, "cuda") / steps
    tokens = wl.SEQS * wl.T
    res.update({"metric": wl.metric, "value": tokens / (ms * 1e-3), "unit": wl.unit, "ms_per_step": ms, "steps": steps,
                "warmup": warmup, "scaling": "strong", "config": wl.config(), "loss": float(wl.out)})
    del wl
    return res


WORKLOADS = {"msda_encoder": MsdaEncoderWorkload, "msda_encoder_bf16": MsdaEncoderBf16Workload,
             "msda_encoder_pairs": MsdaEncoderPairsWorkload, "pair_forward": PairForwardWorkload, "gdino_head": GdinoHeadWorkload,
             "gdino_stage": GdinoStageWorkload, "pair_forward_gdino": PairForwardGdinoWorkload,
             "llm_tp": LlmTpWorkload, "llm_tp_plain": LlmTpPlainWorkload, "internimage_h": InternImageHWorkload, "cfg1_forward": Cfg1Workload,
             "llm_train": LlmTrainWorkload, "llm_tp_train": LlmTpTrainWorkload,
             "pair_forward_1tile": PairForward1TileWorkload, "pair_forward_clip7b": PairForwardClipWorkload,
             "pair_forward_clip7b_1tile": PairForwardClip1TileWorkload, "unipose_stage": UniPoseStageWorkload}
DEFAULT_WORKLOAD = "pair_forward"

# Peak torch.cuda.max_memory_allocated (GB) of `bench.py --gpus 1 --workload NAME` on one NVIDIA H100 80GB HBM3: every
# workload was run there once at the sizes in this file; bench.py repeats the figure in the line's config and reports the
# run's own peak as max_memory_allocated_gb.
H100_80GB_PEAK_GB = {"pair_forward": 65.3, "pair_forward_gdino": 52.4, "pair_forward_1tile": 47.5, "pair_forward_clip7b": 43.0,
                     "pair_forward_clip7b_1tile": 27.4, "llm_train": 55.5, "llm_tp_train": 47.3, "llm_tp": 20.1,
                     "llm_tp_plain": 20.1, "internimage_h": 4.6, "gdino_stage": 3.3, "gdino_head": 1.9, "unipose_stage": 2.9,
                     "cfg1_forward": 0.3, "msda_encoder": 1.2, "msda_encoder_bf16": 1.1, "msda_encoder_pairs": 1.1}


# --------------------------------------------------------------------------------------
# CPU legs: the ONLY place bench code touches oracle/.
# --------------------------------------------------------------------------------------
def _cpu_msda_encoder(steps, warmup):
    import torch
    from oracle import msda_oracle as O
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    value, shapes, lsi, loc, attw = msda_encoder_inputs(torch, 1, torch.device("cpu"), 1234)
    for _ in range(warmup):
        O.forward_grid_sample(value, shapes, loc, attw)
    t0 = time.perf_counter()
    for _ in range(steps):
        O.forward_grid_sample(value, shapes, loc, attw)
    dt = (time.perf_counter() - t0) / steps
    return {"value": 1.0 / dt, "unit": "images/s", "cores": cores, "kind": "port",
            "sample": "1 image per step at the same shape (S=Lq=21760, M=8, D=32, L=4, P=4, fp32), "
                      "oracle.forward_grid_sample = the reference's pure-PyTorch CPU path restated",
            "ms_per_step": dt * 1e3, "sample_ms_per_step": dt * 1e3, "extrapolated": False}


def _cpu_pair_forward_clip(steps, warmup, tiles=5):
    """Reference CPU path of one pair of the released-7B preset, bounded sample: ONE CLIP-L layer on one 336^2 tile (577
    tokens) and ONE Vicuna-7B layer on the T-token sequence, fp32 torch on all host cores (oracle/vit_llm_oracle.py); pair
    time extrapolated as tiles x 24 x t_clip + 32 x t_llm (hidden_states[-2] still runs all 24 layers in HF)."""
    import torch
    from oracle import vit_llm_oracle as VO
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    g = torch.Generator().manual_seed(0)
    C, I, H, F_ = 1024, 4096, 4096, 11008
    T = tiles * 576 + 256
    r = lambda *s: torch.randn(*s, generator=g) * 0.02  # noqa: E731
    csd = {"l.layer_norm1.weight": torch.ones(C), "l.layer_norm1.bias": torch.zeros(C), "l.layer_norm2.weight": torch.ones(C),
           "l.layer_norm2.bias": torch.zeros(C), "l.mlp.fc1.weight": r(I, C), "l.mlp.fc1.bias": torch.zeros(I),
           "l.mlp.fc2.weight": r(C, I), "l.mlp.fc2.bias": torch.zeros(C)}
    for n in ("q", "k", "v", "out"):
        csd[f"l.self_attn.{n}_proj.weight"], csd[f"l.self_attn.{n}_proj.bias"] = r(C, C), torch.zeros(C)
    lsd = {"l.input_layernorm.weight": torch.ones(H), "l.post_attention_layernorm.weight": torch.ones(H),
           "l.self_attn.q_proj.weight": r(H, H), "l.self_attn.k_proj.weight": r(H, H),
           "l.self_attn.v_proj.weight": r(H, H), "l.self_attn.o_proj.weight": r(H, H),
           "l.mlp.gate_proj.weight": r(F_, H), "l.mlp.up_proj.weight": r(F_, H), "l.mlp.down_proj.weight": r(H, F_)}
    xv, xl = torch.randn(1, 577, C, generator=g), torch.randn(1, T, H, generator=g)

    def once():
        t0 = time.perf_counter()
        with torch.no_grad():
            VO.clip_layer(xv, csd, "l.", 16)
        t1 = time.perf_counter()
        with torch.no_grad():
            VO.llama_layer(xl, lsd, "l.", 32, 1e-5)
        return t1 - t0, time.perf_counter() - t1

    for _ in range(warmup):
        once()
    tv = tl = 0.0
    for _ in range(steps):
        a, b = once()
        tv += a; tl += b
    tv /= steps; tl /= steps
    pair_s = tiles * 24 * tv + 32 * tl
    return {"value": 1.0 / pair_s, "unit": "pairs/s", "cores": cores, "kind": "port",
            "sample": f"1 CLIP-L/336 layer x 1 tile ({tv * 1e3:.0f} ms) + 1 Vicuna-7B layer x {T} tokens ({tl * 1e3:.0f} ms), "
                      f"fp32 torch CPU; pair = {tiles * 24} x clip + 32 x llm (extrapolated)",
            "ms_per_step": pair_s * 1e3, "sample_ms_per_step": (tv + tl) * 1e3, "extrapolated": True}


def _cpu_pair_forward(steps, warmup, tiles=5):
    """Reference CPU path of one pair, bounded sample: ONE InternViT-6B layer on one 448^2 tile (1025 tokens) and
    ONE Vicuna-7B layer on the T-token sequence (1536 with 5 tiles), fp32 torch on all host cores
    (oracle/vit_llm_oracle.py); pair time extrapolated as tiles x 48 layers x t_vit + 32 layers x t_llm (embeddings,
    bridge, lm_head left out, so the CPU figure is slightly optimistic)."""
    import torch
    from oracle import vit_llm_oracle as VO
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    g = torch.Generator().manual_seed(0)
    C, I, H, F_ = 3200, 12800, 4096, 11008
    r = lambda *s: torch.randn(*s, generator=g) * 0.02  # noqa: E731
    vsd = {"l.norm1.weight": torch.ones(C), "l.norm2.weight": torch.ones(C), "l.attn.qkv.weight": r(3 * C, C),
           "l.attn.q_norm.weight": torch.ones(C), "l.attn.k_norm.weight": torch.ones(C), "l.attn.proj.weight": r(C, C),
           "l.attn.proj.bias": torch.zeros(C), "l.ls1": torch.full((C,), 0.1), "l.ls2": torch.full((C,), 0.1),
           "l.mlp.fc1.weight": r(I, C), "l.mlp.fc1.bias": torch.zeros(I), "l.mlp.fc2.weight": r(C, I),
           "l.mlp.fc2.bias": torch.zeros(C)}
    lsd = {"l.input_layernorm.weight": torch.ones(H), "l.post_attention_layernorm.weight": torch.ones(H),
           "l.self_attn.q_proj.weight": r(H, H), "l.self_attn.k_proj.weight": r(H, H),
           "l.self_attn.v_proj.weight": r(H, H), "l.self_attn.o_proj.weight": r(H, H),
           "l.mlp.gate_proj.weight": r(F_, H), "l.mlp.up_proj.weight": r(F_, H), "l.mlp.down_proj.weight": r(H, F_)}
    T = tiles * 256 + 256
    xv, xl = torch.randn(1, 1025, C, generator=g), torch.randn(1, T, H, generator=g)

    def once():
        t0 = time.perf_counter()
        with torch.no_grad():
            VO.internvit_layer(xv, vsd, "l.", 25, 1e-6)
        t1 = time.perf_counter()
        with torch.no_grad():
            VO.llama_layer(xl, lsd, "l.", 32, 1e-5)
        return t1 - t0, time.perf_counter() - t1

    for _ in range(warmup):
        once()
    tv = tl = 0.0
    for _ in range(steps):
        a, b = once()
        tv += a; tl += b
    tv /= steps; tl /= steps
    pair_s = tiles * 48 * tv + 32 * tl
    return {"value": 1.0 / pair_s, "unit": "pairs/s", "cores": cores, "kind": "port",
            "sample": f"1 InternViT-6B layer x 1 tile ({tv * 1e3:.0f} ms) + 1 Vicuna-7B layer x {T} tokens "
                      f"({tl * 1e3:.0f} ms), fp32 torch CPU; pair = {tiles * 48} x vit + 32 x llm (extrapolated)",
            "ms_per_step": pair_s * 1e3, "sample_ms_per_step": (tv + tl) * 1e3, "extrapolated": True}


def _cpu_llm_tp(steps, warmup):
    """Reference CPU path of the LLM forward, bounded sample: ONE Vicuna-7B layer on one 2048-token sequence (fp32
    torch, all host cores, oracle/vit_llm_oracle.llama_layer); tokens/s extrapolated over 32 layers (embedding, final
    norm and lm_head left out, so the CPU figure is slightly optimistic)."""
    import torch
    from oracle import vit_llm_oracle as VO
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    g = torch.Generator().manual_seed(0)
    H, F_, T = 4096, 11008, 2048
    r = lambda *s: torch.randn(*s, generator=g) * 0.02  # noqa: E731
    lsd = {"l.input_layernorm.weight": torch.ones(H), "l.post_attention_layernorm.weight": torch.ones(H),
           "l.self_attn.q_proj.weight": r(H, H), "l.self_attn.k_proj.weight": r(H, H),
           "l.self_attn.v_proj.weight": r(H, H), "l.self_attn.o_proj.weight": r(H, H),
           "l.mlp.gate_proj.weight": r(F_, H), "l.mlp.up_proj.weight": r(F_, H), "l.mlp.down_proj.weight": r(H, F_)}
    x = torch.randn(1, T, H, generator=g)
    for _ in range(warmup):
        with torch.no_grad():
            VO.llama_layer(x, lsd, "l.", 32, 1e-5)
    t0 = time.perf_counter()
    for _ in range(steps):
        with torch.no_grad():
            VO.llama_layer(x, lsd, "l.", 32, 1e-5)
    tl = (time.perf_counter() - t0) / steps
    seq_s = 32 * tl
    return {"value": T / seq_s, "unit": "tokens/s", "cores": cores, "kind": "port",
            "sample": f"1 Vicuna-7B layer x one 2048-token sequence ({tl * 1e3:.0f} ms), fp32 torch CPU; "
                      "sequence = 32 x layer (extrapolated)",
            "ms_per_step": 8 * seq_s * 1e3, "sample_ms_per_step": tl * 1e3, "extrapolated": True}


def _cpu_internimage_h(steps, warmup):
    """Reference CPU path of the InternImage-H backbone, bounded sample: ONE level-0 layer (320 channels, 10 groups,
    5x5 depthwise branch, DCNv3 core through the C oracle = the reference CUDA kernel's arithmetic restated, fp32 torch
    for the projections / MLP / norms) on one 256x256 map; an image is extrapolated as 50 such layers (every level's
    layer costs the same FLOPs: a quarter of the pixels at twice the width), stem and downsampling left out."""
    import numpy as np
    import torch
    import torch.nn.functional as F
    from oracle import dcnv3_oracle as O
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    g = torch.Generator().manual_seed(0)
    C, G, K, Hh = 320, 10, 9, 256
    r = lambda *s: torch.randn(*s, generator=g) * 0.02  # noqa: E731
    x = torch.randn(1, Hh, Hh, C, generator=g)
    w_in, w_out, w_dw, w_off, w_mask = r(C, C), r(C, C), r(C, 1, 5, 5), r(G * K * 2, C), r(G * K, C)
    w1, w2 = r(4 * C, C), r(C, 4 * C)

    def once():
        t0 = time.perf_counter()
        with torch.no_grad():
            h = F.layer_norm(x, (C,))
            xp = F.linear(h, w_in)
            x1 = F.gelu(F.layer_norm(F.conv2d(h.permute(0, 3, 1, 2), w_dw, padding=2, groups=C).permute(0, 2, 3, 1), (C,)))
            off = F.linear(x1, w_off).contiguous()
            msk = F.softmax(F.linear(x1, w_mask).view(1, Hh, Hh, G, K), -1).reshape(1, Hh, Hh, G * K).contiguous()
            core = torch.from_numpy(np.asarray(O.forward(xp.numpy(), off.numpy(), msk.numpy(), 3, 3, 1, 1, 1, 1, 1, 1, G,
                                                         C // G, 1.0), dtype=np.float32))
            y = x + F.layer_norm(F.linear(core, w_out), (C,))
            y = y + F.layer_norm(F.linear(F.gelu(F.linear(F.layer_norm(y, (C,)), w1)), w2), (C,))
        return time.perf_counter() - t0

    for _ in range(warmup):
        once()
    tl = sum(once() for _ in range(steps)) / steps
    img_s = 50 * tl
    return {"value": 1.0 / img_s, "unit": "images/s", "cores": cores, "kind": "port",
            "sample": f"1 level-0 InternImage-H layer on one 256x256x320 map ({tl * 1e3:.0f} ms; DCNv3 core = C oracle, "
                      "projections fp32 torch); image = 50 x layer (extrapolated)",
            "ms_per_step": 4 * img_s * 1e3, "sample_ms_per_step": tl * 1e3, "extrapolated": True}


def _cpu_cfg1(steps, warmup):
    """BASELINE cfg 1's "CPU reference fwd", MEASURED (not extrapolated): the same module graph as the GPU arm with
    every kernel replaced by its fp32 torch stand-in (oracle/torch_kernels.py; MSDA = the reference's pure-PyTorch
    grid_sample fallback restated) on the host cores.  tests/test_cfg1_logic_cpu.py pins this port to the reference's own
    modules (1e-6).  The golden also records the reference modules' own CPU time in the build container."""
    import numpy as np
    import torch
    from oracle import torch_kernels as TK
    C = Cfg1Workload._common()
    cores = min(os.cpu_count() or 1, 32)
    torch.set_num_threads(cores)
    model = C.build_b200_model(None, device="cpu", dtype=torch.float32)
    ids, image, aug = C.inputs()
    mask = torch.ones_like(ids)

    def once():
        with TK.patched():
            model(input_ids=ids, attention_mask=mask, images=image, images_aug=[aug[0]], img_metas=[{"task": "det"}])

    for _ in range(warmup):
        once()
    t0 = time.perf_counter()
    for _ in range(steps):
        once()
    dt = (time.perf_counter() - t0) / steps
    ref_ms = None
    try:
        ref_ms = float(np.load(os.path.join(ROOT, "tests", "golden", "cfg1_e2e.npz"))["cpu_ms_fp32_8threads"])
    except Exception:
        pass
    return {"value": 1.0 / dt, "unit": "pairs/s", "cores": cores, "kind": "port", "extrapolated": False,
            "sample": "the whole cfg-1 forward, 1 pair per step, fp32 torch CPU (kernels -> oracle/torch_kernels.py stand-ins)",
            "ms_per_step": dt * 1e3, "sample_ms_per_step": dt * 1e3, "steps_run": steps,
            "reference_modules_cpu_ms_in_build_container_8_threads": ref_ms}


def _cpu_llm_train(steps, warmup):
    """Reference CPU path of the fwd+bwd step, bounded sample: ONE Vicuna-7B layer on one 2048-token sequence, torch fp32
    autograd on all host cores (oracle/vit_llm_oracle.llama_layer, sum-of-outputs loss); tokens/s extrapolated over 32 layers."""
    import torch
    from oracle import vit_llm_oracle as VO
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    g = torch.Generator().manual_seed(0)
    H, F_, T = 4096, 11008, 2048
    r = lambda *s: (torch.randn(*s, generator=g) * 0.02).requires_grad_(True)  # noqa: E731
    lsd = {"l.input_layernorm.weight": torch.ones(H, requires_grad=True), "l.post_attention_layernorm.weight": torch.ones(H, requires_grad=True),
           "l.self_attn.q_proj.weight": r(H, H), "l.self_attn.k_proj.weight": r(H, H),
           "l.self_attn.v_proj.weight": r(H, H), "l.self_attn.o_proj.weight": r(H, H),
           "l.mlp.gate_proj.weight": r(F_, H), "l.mlp.up_proj.weight": r(F_, H), "l.mlp.down_proj.weight": r(H, F_)}
    x = torch.randn(1, T, H, generator=g).requires_grad_(True)

    def once():
        for t in list(lsd.values()) + [x]:
            t.grad = None
        VO.llama_layer(x, lsd, "l.", 32, 1e-5).sum().backward()

    for _ in range(warmup):
        once()
    t0 = time.perf_counter()
    for _ in range(steps):
        once()
    tl = (time.perf_counter() - t0) / steps
    return {"value": T / (32 * tl), "unit": "tokens/s", "cores": cores, "kind": "port",
            "sample": f"1 Vicuna-7B layer fwd+bwd x one 2048-token sequence ({tl * 1e3:.0f} ms), fp32 torch CPU autograd; "
                      "sequence = 32 x layer (extrapolated)",
            "ms_per_step": 4 * 32 * tl * 1e3, "sample_ms_per_step": tl * 1e3, "extrapolated": True}


_CPU = {"msda_encoder": _cpu_msda_encoder, "msda_encoder_bf16": _cpu_msda_encoder, "msda_encoder_pairs": _cpu_msda_encoder, "pair_forward": _cpu_pair_forward, "gdino_head": _cpu_msda_encoder,
        "gdino_stage": _cpu_msda_encoder,
        "pair_forward_gdino": _cpu_pair_forward, "llm_tp": _cpu_llm_tp, "llm_tp_plain": _cpu_llm_tp, "internimage_h": _cpu_internimage_h, "cfg1_forward": _cpu_cfg1, "llm_train": _cpu_llm_train,
        "llm_tp_train": _cpu_llm_train,
        "pair_forward_1tile": lambda steps, warmup: _cpu_pair_forward(steps, warmup, tiles=1),
        "pair_forward_clip7b": _cpu_pair_forward_clip,
        "pair_forward_clip7b_1tile": lambda steps, warmup: _cpu_pair_forward_clip(steps, warmup, tiles=1),
        "unipose_stage": _cpu_msda_encoder}


def cpu_baseline(name):
    return _CPU[name](steps=3, warmup=1)


def run_reference_arm(name, n_gpus, steps, warmup):
    """`bench.py --impl reference`: the CPU port of the path on the host cores.  For the full-size workloads a step is
    a BOUNDED SAMPLE (one layer of each tower at real width) and the workload figure is EXTRAPOLATED from it -- the
    line says so (`extrapolated`, `sample_ms_per_step`, `steps` = sample steps really run); cfg 1 is measured whole."""
    wl = WORKLOADS[name]
    run_steps = max(1, min(steps, 20 if name == "cfg1_forward" else 5))
    run_warm = max(1, min(warmup, 2))
    t0 = time.perf_counter()
    cb = _CPU[name](steps=run_steps, warmup=run_warm)
    wall = time.perf_counter() - t0
    cb.setdefault("extrapolated", True)
    cb["steps_run"] = run_steps
    return {"impl": "reference", "metric": wl.metric, "value": cb["value"], "unit": wl.unit, "n_gpus": n_gpus,
            "steps": run_steps, "steps_requested": steps, "warmup": run_warm, "ms_per_step": cb["ms_per_step"],
            "extrapolated": cb["extrapolated"], "sample_ms_per_step": cb.get("sample_ms_per_step"), "wall_s": wall,
            "higher_is_better": True,
            "scaling": "strong" if name in ("llm_tp", "llm_tp_plain", "llm_tp_train") else "weak", "vs_baseline": None,
            "dtype": "f32 (torch CPU; the GPU arm computes in " + wl.dtype + ")",
            "data": "synthetic", "config": {"workload": cb["sample"]}, "cpu_baseline": cb,
            "e2e": {"value": cb["value"], "unit": wl.unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
