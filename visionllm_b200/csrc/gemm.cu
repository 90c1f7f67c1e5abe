// bf16 GEMM with fused epilogue on the sm_90a tensor cores (wgmma + TMA + mbarrier).
//
//   C[M, N] = epilogue( A[M, K] . B[N, K]^T )      A, B bf16 K-major (B is an nn.Linear weight [out, in])
//   epilogue: (+bias[N]) -> act -> (*colscale[N]) -> (+residual[M, N]) -> bf16 | fp32
//   act = SWIGLU pairs columns (2j, 2j+1) = (gate_j, up_j) and writes N/2 columns.
//
// This one kernel carries every dense projection on the hot path (SURVEY.md 8a / Appendix B):
//   InternViT  qkv / proj(+bias, *ls1, +x) / fc1(+bias, GELU) / fc2(+bias, *ls2, +x)
//              (internvit/modeling_intern_vit.py:112,124,172-173,206-208), patch-embed as im2col GEMM (:73-85)
//   vl_bridge  Linear+GELU+Linear (modeling_visionllmv2.py:162-184)
//   LLM        q/k/v/o, gate|up (SwiGLU), down(+residual)  (HF LlamaDecoderLayer; internlm2/modeling_internlm2.py:235-360)
//   GDINO      value/offset/weight/output projections, FFN (ReLU)  (grounding_dino/...mask_dn.py:674-677,1116-1117)
//
// Structure (persistent, warp-specialised, one CTA of three warpgroups per SM):
//   warpgroup 0    producer: one elected lane of warp 0 issues the TMA loads, A tile 128x64 and B tile (256|128)x64
//                  bf16, 128B swizzle, STAGES-deep mbarrier ring; the warpgroup hands its registers to the consumers
//   warpgroups 1-2 consumers: warpgroup w owns rows 64(w-1)..64(w-1)+63 of the tile and issues wgmma m64n128k16
//                  (one or two per k-step) straight from the swizzled stages; fp32 accumulators stay in registers
//                  (64 x BN / 128 threads = 64 | 128 per thread).  One k-block of MMAs stays in flight while the next
//                  stage is awaited; a stage goes back to the producer when the MMAs that read it have retired.
//                  The fused epilogue runs on the accumulator fragments (a thread owns column pairs of two rows, so
//                  the SwiGLU (gate, up) pair never leaves a thread); bf16 output is staged per warp in shared memory
//                  and leaves as 128-byte row runs; the producer keeps prefetching the next tile's stages meanwhile.
// Tiles are visited in groups of GROUP_M row-blocks so concurrently running CTAs share B (weights) in L2.
#include "common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int BM = 128, BK = 64, THREADS = 384, CONSUMER_WARPS = 8, CONSUMER_THREADS = CONSUMER_WARPS * 32;
constexpr int A_BYTES = BM * BK * 2;
constexpr int EPI_PITCH = 128 + 16;                 // 64 bf16 columns + 16 B pad: conflict-free fragment writes and 16-byte reads
constexpr int EPI_WARP_BYTES = 16 * EPI_PITCH;      // a consumer warp's 16 rows of one 64-column chunk

enum { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2, ACT_SILU = 3, ACT_SWIGLU = 4, ACT_QUICKGELU = 5 };

struct GemmArgs {
  int M, N, K;
  void* C; int ldc;
  const __nv_bfloat16* bias; const __nv_bfloat16* colscale; const __nv_bfloat16* residual; int ldr;
  int act; int out_f32;
  const unsigned char* row_keep;   // optional [M]: rows with 0 are written as exact zeros (value.masked_fill of the MSDA module)
  int tiles_m, tiles_n;
  int group_m;           // row-blocks per rasterisation group (see pick_group_m)
  // Implicit convolution over a zero-padded channels-last image (vllm_conv_rows_bf16): the K axis is a_segs segments
  // of a_seg_kb k-blocks; segment s reads A rows shifted by s * a_seg_rows (one image row of the padded map), and a
  // row of the A tensor map spans kw consecutive pixels (row pitch = C elements, row length = kw*C: rows overlap).
  int a_seg_kb, a_seg_rows;
  // Fused reduce-scatter push (vllm_gemm_bf16_scatter, tensor-parallel o_proj): row block d = row / sc_rows of C goes
  // to sc_dst[d] (a peer GPU's receive slot, row pitch ldc, local row = row - d * sc_rows); every consumer warp bumps
  // sc_flag[d] once per tile after its stores (release at system scope).  sc_rows == 0: plain GEMM.
  int sc_rows;
  void* sc_dst[8];
  uint32_t* sc_flag[8];
  // MN-major operands (vllm_gemm_bf16_tn: the backward GEMMs -- dgrad reads the nn.Linear weight [N_red, K_out] as
  // B[j, k] = W[k, j], wgrad reads grad_output / activations [tokens, features] with the token axis as K): the operand
  // is a row-major [K, MN] matrix; a 64-k x 64-mn TMA box is one 128B-swizzled MN-major wgmma atom row, chunks of 64 mn
  // are 8 KB apart in the stage (LBO), 8 k-rows 1 KB apart (SBO), a k-step of 16 advances 2 KB.
  int a_mn, b_mn;
  // Block-diagonal batching (vllm_gemm_bf16_batched: the attention-backward GEMMs over all (batch, head) matrices of a
  // layer in one launch): every operand is a stack of `bt_rows`-row matrices along its row axis; the output row block
  // m0 belongs to matrix m0 / bt_rows and only meets that matrix's B rows / K range.  causal: 1 = skip output tiles
  // strictly above the diagonal (S = Q K^T, dP = dO V^T), 2 = the K range starts at the tile's first row (dV = P^T dO,
  // dK = dS^T Q: P, dS are zero below), 3 = the K range ends at the tile's last row (dQ = dS K).
  int bt_rows, causal;
};

// per-tile K range / operand offsets of the batched mode (identity when bt_rows == 0)
struct TilePlan { int skip, kb0, kb1, b_row_off, k_off; };
__device__ __forceinline__ TilePlan plan_tile(const GemmArgs& g, int m0, int n0, int rows_per_tile, int num_kb) {
  TilePlan p{0, 0, num_kb, 0, 0};
  if (g.bt_rows) {
    const int bh = m0 / g.bt_rows, ml = m0 - bh * g.bt_rows;
    p.b_row_off = bh * g.N;                             // K-major B: a stack of [N, K] matrices along the rows
    p.k_off = bh * g.K;                                 // MN-major operands: stacks of [K, M|N] matrices along the K rows
    if (g.causal == 1 && n0 >= ml + rows_per_tile) p.skip = 1;
    if (g.causal == 2) p.kb0 = ml / BK;
    if (g.causal == 3) { const int e = (ml + rows_per_tile + BK - 1) / BK; p.kb1 = e < num_kb ? e : num_kb; }
  }
  return p;
}

template <int BN> struct Cfg {
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 256 ? 4 : 6;     // 192 KB of operand stages either way
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + 2 * BN * 4 /*bias, scale*/ +
                              CONSUMER_WARPS * EPI_WARP_BYTES /*per-warp store staging*/;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& tm, int& tn) {
  const int per_group = group_m * tiles_n;
  const int group = t / per_group;
  const int first = group * group_m;
  const int gsz = min(group_m, tiles_m - first);
  const int in = t - group * per_group;
  tm = first + in % gsz;
  tn = in / gsz;
}

// the four operand-layout combinations of one k-block (BK = 4 k-steps) of a warpgroup's 64 x BN tile
template <int TA, int TB, int NB>
__device__ __forceinline__ void mma_kblock(float (&acc)[NB][64], uint32_t sa, uint32_t sb, bool first_kb) {
  // K-major: a k-step of 16 bf16 advances the start address by 32 B inside the 128 B swizzle row;
  // MN-major: by 16 k-rows x 128 B = 2 KB (descriptor address units are 16 B)
  const uint64_t adesc = TA ? tc::wgmma_desc_sw128(sa, 8192, 1024) : tc::wgmma_desc_sw128(sa, 16, 1024);
  const uint64_t bdesc = TB ? tc::wgmma_desc_sw128(sb, 8192, 1024) : tc::wgmma_desc_sw128(sb, 16, 1024);
  constexpr uint64_t astep = TA ? 128 : 2, bstep = TB ? 128 : 2;
  constexpr uint64_t bhalf = 16384 >> 4;     // columns 128.. of the B tile: 128 K-major rows or two MN-major chunks
#pragma unroll
  for (int k = 0; k < BK / 16; ++k)
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
      tc::wgmma_m64n128k16_ss<TA, TB>(acc[nb], adesc + astep * k, bdesc + bstep * k + bhalf * nb, !(first_kb && k == 0));
}

template <int BN>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmArgs g) {
  using C_ = Cfg<BN>;
  constexpr int STAGES = C_::STAGES, NB = BN / 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - tc::smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + STAGES * C_::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8 * s; };
  auto empty_bar = [&](int s) { return bar_base + 8 * (STAGES + s); };
  float* s_bias = reinterpret_cast<float*>(smem_gen + STAGES * C_::STAGE_BYTES + 256);
  float* s_scale = s_bias + BN;
  uint8_t* s_epi = reinterpret_cast<uint8_t*>(s_scale + BN);   // CONSUMER_WARPS x 16 rows x EPI_PITCH bytes

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = g.tiles_m * g.tiles_n;
  const int num_kb = (g.K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    tc::tma_prefetch_desc(&tmap_a);
    tc::tma_prefetch_desc(&tmap_b);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), CONSUMER_WARPS); }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    tc::reg_dealloc<40>();
    if (warp == 0 && tc::elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        int tm, tn; tile_coords(t, g.tiles_m, g.tiles_n, g.group_m, tm, tn);
        const TilePlan tp = plan_tile(g, tm * BM, tn * BN, BM, num_kb);
        if (tp.skip) continue;
        const int bt_m0 = g.bt_rows ? (tm * BM) / g.bt_rows * g.bt_rows : 0;
        // K-major A: global stacked row; MN-major A: column inside its matrix (the stack runs along the K rows)
        const int row_a = tm * BM - (g.a_mn ? bt_m0 : 0);
        const int row_b = tn * BN + (g.b_mn ? 0 : tp.b_row_off);
        const int ka_off = g.a_mn ? tp.k_off : 0, kb_off = g.b_mn ? tp.k_off : 0;
        for (int kb = tp.kb0; kb < tp.kb1; ++kb) {
          tc::mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * C_::STAGE_BYTES, sb = sa + A_BYTES;
          int ka = kb * BK + ka_off, ra = row_a;
          if (g.a_seg_kb) {
            const int seg = kb / g.a_seg_kb;
            ka = (kb - seg * g.a_seg_kb) * BK;
            ra = row_a + seg * g.a_seg_rows;
          }
          tc::mbar_arrive_expect_tx(full_bar(stage), C_::STAGE_BYTES);
          if (g.a_mn) {
            for (int h = 0; h < BM / 64; ++h) tc::tma_load_2d(sa + h * 8192, &tmap_a, full_bar(stage), ra + 64 * h, ka);
          } else {
            tc::tma_load_2d(sa, &tmap_a, full_bar(stage), ka, ra);
          }
          if (g.b_mn) {
            for (int h = 0; h < BN / 64; ++h)
              tc::tma_load_2d(sb + h * 8192, &tmap_b, full_bar(stage), row_b + 64 * h, kb * BK + kb_off);
          } else {
            tc::tma_load_2d(sb, &tmap_b, full_bar(stage), kb * BK, row_b);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: main loop + epilogue =====================
  tc::reg_alloc<232>();
  const int wg = (warp - 4) >> 2;                  // 0 / 1: rows 0-63 / 64-127 of the tile
  const int et = threadIdx.x - 128;                // 0..255
  const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2), frag_col = 2 * (lane & 3);
  const bool swiglu = g.act == ACT_SWIGLU;
  int stage = 0; uint32_t phase = 0;
  float acc[NB][64];
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    int tm, tn; tile_coords(t, g.tiles_m, g.tiles_n, g.group_m, tm, tn);
    const TilePlan tp = plan_tile(g, tm * BM, tn * BN, BM, num_kb);
    if (tp.skip) continue;
    const int n0 = tn * BN;
    // bias / column scale of the tile go to shared memory now (broadcast reads in the epilogue math), so their global-load
    // latency hides under the main loop; the previous tile's readers left at the barrier that closed its epilogue
    if (et < BN) {
      const int col = n0 + et;
      s_bias[et] = (g.bias && col < g.N) ? __bfloat162float(g.bias[col]) : 0.f;
      s_scale[et] = (g.colscale && col < g.N) ? __bfloat162float(g.colscale[col]) : 1.f;
    }
    int prev_stage = -1;
    for (int kb = tp.kb0; kb < tp.kb1; ++kb) {
      tc::mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * C_::STAGE_BYTES + wg * 8192, sb = smem_base + stage * C_::STAGE_BYTES + A_BYTES;
      const bool first = kb == tp.kb0;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) tc::acc_fence(acc[nb]);
      tc::wgmma_fence();
      if (g.a_mn) {
        if (g.b_mn) mma_kblock<1, 1, NB>(acc, sa, sb, first); else mma_kblock<1, 0, NB>(acc, sa, sb, first);
      } else {
        if (g.b_mn) mma_kblock<0, 1, NB>(acc, sa, sb, first); else mma_kblock<0, 0, NB>(acc, sa, sb, first);
      }
      tc::wgmma_commit();
      tc::wgmma_wait<1>();                           // the previous k-block's MMAs have retired: its stage is free
      if (prev_stage >= 0 && lane == 0) tc::mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    tc::wgmma_wait<0>();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) tc::acc_fence(acc[nb]);
    if (lane == 0) tc::mbar_arrive(empty_bar(prev_stage));
    tc::named_bar_sync(1, CONSUMER_THREADS);         // s_bias / s_scale of this tile are in place

    // ---- epilogue on the accumulator fragments: element pair (c, c + 1) of rows r and r + 8 per n8 block ----
    // bias -> activation -> column scale -> residual -> row mask on the pair (c, c + 1) of `row` (not for SwiGLU)
    auto math = [&](int row, int c, float& v0, float& v1) {
      const int col = n0 + c;
      v0 += s_bias[c]; v1 += s_bias[c + 1];
      if (g.act == ACT_GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
      else if (g.act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      else if (g.act == ACT_SILU) { v0 = silu(v0); v1 = silu(v1); }
      else if (g.act == ACT_QUICKGELU) { v0 = v0 / (1.f + __expf(-1.702f * v0)); v1 = v1 / (1.f + __expf(-1.702f * v1)); }
      v0 *= s_scale[c]; v1 *= s_scale[c + 1];
      if (row >= g.M) return;
      if (g.residual) {
        const __nv_bfloat16* rp = g.residual + (size_t)row * g.ldr + col;
        if (col + 1 < g.N) {                         // col is even: a pair is 4-byte aligned
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(rp));
          v0 += f.x; v1 += f.y;
        } else {
          v0 += __bfloat162float(rp[0]);
        }
      }
      if (g.row_keep && !g.row_keep[row]) { v0 = 0.f; v1 = 0.f; }
    };
    // destination of an output row: C, or the peer slot that owns row block d of C (scatter mode)
    auto out_row = [&](int row) -> __nv_bfloat16* {
      if (!g.sc_rows) return reinterpret_cast<__nv_bfloat16*>(g.C) + (size_t)row * g.ldc;
      const int d = row / g.sc_rows;
      return reinterpret_cast<__nv_bfloat16*>(g.sc_dst[d]) + (size_t)(row - d * g.sc_rows) * g.ldc;
    };
    // general path: the pair goes straight from the fragment to global memory (fp32 output, SwiGLU, ragged N)
    auto emit = [&](int row, int c, float v0, float v1) {
      const int col = n0 + c;
      if (row >= g.M || col >= g.N) return;
      if (swiglu) {                                  // columns (2j, 2j+1) = (gate, up) -> output column j
        const int oc = col >> 1;
        float o = silu(v0 + s_bias[c]) * (v1 + s_bias[c + 1]);
        if (g.residual) o += __bfloat162float(g.residual[(size_t)row * g.ldr + oc]);
        reinterpret_cast<__nv_bfloat16*>(g.C)[(size_t)row * g.ldc + oc] = __float2bfloat16(o);
        return;
      }
      math(row, c, v0, v1);
      const bool pair = col + 1 < g.N;               // 4-byte (bf16) / 8-byte (fp32) aligned
      if (g.out_f32) {
        float* cp = reinterpret_cast<float*>(g.C) + (size_t)row * g.ldc + col;
        if (pair) *reinterpret_cast<float2*>(cp) = make_float2(v0, v1); else cp[0] = v0;
        return;
      }
      __nv_bfloat16* cp = out_row(row) + col;
      if (pair) *reinterpret_cast<__nv_bfloat162*>(cp) = __floats2bfloat162_rn(v0, v1); else cp[0] = __float2bfloat16(v0);
    };
    const int row0 = tm * BM + frag_row;
    const int warp_row0 = tm * BM + wg * 64 + (warp & 3) * 16;
    uint8_t* my_stage = s_epi + (warp - 4) * EPI_WARP_BYTES;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {               // 64-column chunks of this 128-column accumulator half
        const int c0 = nb * 128 + ch * 64;
        if (n0 + c0 >= g.N) break;                   // uniform
        if (swiglu || g.out_f32 || n0 + c0 + 64 > g.N) {
#pragma unroll
          for (int j = 8 * ch; j < 8 * ch + 8; ++j) {
            const int c = nb * 128 + 8 * j + frag_col;
            emit(row0, c, acc[nb][4 * j], acc[nb][4 * j + 1]);
            emit(row0 + 8, c, acc[nb][4 * j + 2], acc[nb][4 * j + 3]);
          }
          continue;
        }
        // bf16 fast path: the warp stages its 16 rows x 64 columns in shared memory, then stores 128-byte row runs
        // (4-byte stores from the fragments would cost the L2 eight requests per 128-byte line instead of one)
#pragma unroll
        for (int j = 8 * ch; j < 8 * ch + 8; ++j) {
          const int c = nb * 128 + 8 * j + frag_col;
          float a0 = acc[nb][4 * j], a1 = acc[nb][4 * j + 1], b0 = acc[nb][4 * j + 2], b1 = acc[nb][4 * j + 3];
          math(row0, c, a0, a1);
          math(row0 + 8, c, b0, b1);
          const int off = (8 * (j - 8 * ch) + frag_col) * 2;
          *reinterpret_cast<__nv_bfloat162*>(my_stage + (lane >> 2) * EPI_PITCH + off) = __floats2bfloat162_rn(a0, a1);
          *reinterpret_cast<__nv_bfloat162*>(my_stage + ((lane >> 2) + 8) * EPI_PITCH + off) = __floats2bfloat162_rn(b0, b1);
        }
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 4; ++it) {             // each instruction: 4 rows x 128 contiguous bytes
          const int rr = it * 4 + (lane >> 3), piece = lane & 7;
          const uint4 val = *reinterpret_cast<const uint4*>(my_stage + rr * EPI_PITCH + piece * 16);
          if (warp_row0 + rr < g.M) *reinterpret_cast<uint4*>(out_row(warp_row0 + rr) + n0 + c0 + piece * 8) = val;
        }
        __syncwarp();
      }
    }
    if (g.sc_rows) {                                 // tile pushed: publish it to the owner of these rows
      __threadfence_system();
      __syncwarp();
      if (lane == 0 && warp_row0 < g.M)
        asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(g.sc_flag[warp_row0 / g.sc_rows]), "r"(1u) : "memory");
    }
    tc::named_bar_sync(1, CONSUMER_THREADS);         // every reader of s_bias / s_scale is done: the next tile may overwrite
  }
}

// Rasterisation: a group of `group_m` row-blocks sweeps all column-blocks before the next group starts, so one wave of
// CTAs covers a near-square patch of tiles (minimal A+B bytes per wave).  The knob remains for sweeps.
int g_group_m_override = 0;
// SM budgets (0 = every SM): a persistent GEMM CTA owns its SM (384 threads with the whole register file between them), so a
// link-bound kernel of another stream -- the peer pushes of the tensor-parallel exchange -- can only overlap a GEMM on SMs
// the GEMM's grid leaves free.  g_sm_limit caps every launch, g_scatter_sm_limit the scatter GEMM (vllm_gemm_bf16_scatter),
// whose epilogue stores ride NVLink while the other micro-batch's GEMM runs beside it (visionllm_b200/tp.py).
int g_sm_limit = 0, g_scatter_sm_limit = 0;
int pick_group_m(int, int, long long) { return g_group_m_override > 0 ? g_group_m_override : 8; }

// 0: auto = 128 x 128 tiles (faster than 128 x 256 at every hot-path shape measured on an H100, README.md);
// 1 / 2: force the 128- / 256-column tile (tests and sweeps).  The scatter GEMM always uses 128 x 256: its receivers
// count arrivals per such tile.
int g_gemm_variant = 0;

template <int BN>
int launch_gemm(const void* A, int lda, const void* B, int ldb, GemmArgs g, cudaStream_t st, long long a_rows = -1,
                int a_cols = -1) {
  using C_ = Cfg<BN>;
  CUtensorMap ta, tb;
  const uint64_t nb = g.bt_rows ? (uint64_t)(g.M / g.bt_rows) : 1;     // matrices in the stack (batched mode)
  const uint64_t m_local = g.bt_rows ? (uint64_t)g.bt_rows : (uint64_t)g.M;
  int rc = g.a_mn ? vllm_make_tmap_bf16(&ta, A, nb * (uint64_t)g.K, m_local, (uint64_t)lda, 64)       // [K, M] rows, 64 x 64 boxes
                  : vllm_make_tmap_bf16(&ta, A, (uint64_t)(a_rows < 0 ? g.M : a_rows),
                                        (uint64_t)(a_cols < 0 ? g.K : a_cols), (uint64_t)lda, BM);
  if (rc) return rc;
  rc = g.b_mn ? vllm_make_tmap_bf16(&tb, B, nb * (uint64_t)g.K, (uint64_t)g.N, (uint64_t)ldb, 64)
              : vllm_make_tmap_bf16(&tb, B, nb * (uint64_t)g.N, (uint64_t)g.K, (uint64_t)ldb, BN);
  if (rc) return rc;
  g.tiles_m = (g.M + BM - 1) / BM;
  g.tiles_n = (g.N + BN - 1) / BN;
  const int n_tiles = g.tiles_m * g.tiles_n;
  int sms = vllm_num_sms();
  const int limit = g.sc_rows ? (g_scatter_sm_limit > 0 ? g_scatter_sm_limit : g_sm_limit) : g_sm_limit;
  if (limit > 0 && limit < sms) sms = limit;
  const int ctas = sms < n_tiles ? sms : n_tiles;
  g.group_m = pick_group_m(sms, g.tiles_n, (long long)g.N * g.K * 2);
  static bool attr_set[64] = {false};
  bool* set = vllm_device_flag(attr_set);
  if (!set || !*set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C_::SMEM);
    if (e != cudaSuccess) return (int)e;
    if (set) *set = true;
  }
  gemm_bf16_wgmma_kernel<BN><<<ctas, THREADS, C_::SMEM, st>>>(ta, tb, g);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int launch_gemm_auto(const void* A, int lda, const void* B, int ldb, const GemmArgs& g, cudaStream_t st, long long a_rows = -1,
                     int a_cols = -1) {
  // the receivers of a scatter GEMM count 8 arrivals per 128 x 256 tile (visionllm_b200/tp.py)
  const bool wide = g.sc_rows || g_gemm_variant == 2;
  return wide ? launch_gemm<256>(A, lda, B, ldb, g, st, a_rows, a_cols) : launch_gemm<128>(A, lda, B, ldb, g, st, a_rows, a_cols);
}

}  // namespace

extern "C" {

int vllm_gemm_set_variant(int v) { g_gemm_variant = (v == 1 || v == 2) ? v : 0; return VLLM_OK; }
int vllm_gemm_set_group_m(int gm) { g_group_m_override = gm; return VLLM_OK; }
int vllm_gemm_set_sm_limit(int all_gemms, int scatter_gemm) {
  if (all_gemms < 0 || scatter_gemm < 0) return VLLM_EINVAL;
  g_sm_limit = all_gemms; g_scatter_sm_limit = scatter_gemm;
  return VLLM_OK;
}

static int gemm_bf16_common(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                            const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                            const unsigned char* row_keep, void* stream);

int vllm_gemm_bf16(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                   const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                   void* stream) {
  return gemm_bf16_common(A, lda, B, ldb, C, ldc, M, N, K, bias, colscale, residual, ldr, act, out_f32, nullptr, stream);
}

int vllm_gemm_bf16_rowmask(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                           const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                           const unsigned char* row_keep, void* stream) {
  if (!row_keep || act == ACT_SWIGLU) return VLLM_EINVAL;
  return gemm_bf16_common(A, lda, B, ldb, C, ldc, M, N, K, bias, colscale, residual, ldr, act, out_f32, row_keep, stream);
}

static int gemm_bf16_common(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                            const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                            const unsigned char* row_keep, void* stream) {
  if (M < 0 || N <= 0 || K <= 0 || lda < K || ldb < K) return VLLM_EINVAL;
  if (M == 0) return VLLM_OK;
  if (!A || !B || !C) return VLLM_EINVAL;
  if (act < 0 || act > ACT_QUICKGELU) return VLLM_EINVAL;
  const int n_out = act == ACT_SWIGLU ? N / 2 : N;
  if (act == ACT_SWIGLU && (N % 2 || out_f32 || colscale)) return VLLM_EUNSUPPORTED;
  if (ldc < n_out || (residual && ldr < n_out)) return VLLM_EINVAL;
  // TMA: 16-byte aligned bases and row pitches; vector epilogue: 16-byte aligned rows
  if (!vllm_aligned(A, 16) || !vllm_aligned(B, 16) || (lda % 8) || (ldb % 8)) return VLLM_EALIGN;
  const int celt = out_f32 ? 4 : 2;
  if (!vllm_aligned(C, 16) || ((size_t)ldc * celt) % 16 || (residual && (!vllm_aligned(residual, 16) || ldr % 8)))
    return VLLM_EALIGN;
  GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.C = C; g.ldc = ldc;
  g.bias = (const __nv_bfloat16*)bias; g.colscale = (const __nv_bfloat16*)colscale;
  g.residual = (const __nv_bfloat16*)residual; g.ldr = ldr; g.act = act; g.out_f32 = out_f32;
  g.row_keep = row_keep;
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(A, lda, B, ldb, g, st);
}

int vllm_gemm_bf16_tn(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C, int ldc, int M,
                      int N, int K, int out_f32, void* stream) {
  // C[M, N] = sum_k A(m, k) * B(n, k) with either operand stored K-major ([rows = M|N, cols = K], like vllm_gemm_bf16) or
  // MN-major ([rows = K, cols = M|N], pitch lda / ldb): the backward GEMMs of a Linear y = x W^T without transposed copies --
  //   dgrad  dx[T, in]  = dy[T, out] (K-major A, K = out) x W[out, in] as MN-major B
  //   wgrad  dW[out, in] = dy[T, out] as MN-major A (K = T) x x[T, in] as MN-major B.
  if (M < 0 || N <= 0 || K <= 0) return VLLM_EINVAL;
  if (M == 0) return VLLM_OK;
  if (!A || !B || !C) return VLLM_EINVAL;
  if (lda < (a_mn_major ? M : K) || ldb < (b_mn_major ? N : K) || ldc < N) return VLLM_EINVAL;
  if (!vllm_aligned(A, 16) || !vllm_aligned(B, 16) || (lda % 8) || (ldb % 8)) return VLLM_EALIGN;
  if (!vllm_aligned(C, 16) || ((size_t)ldc * (out_f32 ? 4 : 2)) % 16) return VLLM_EALIGN;
  GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.C = C; g.ldc = ldc; g.out_f32 = out_f32;
  g.a_mn = a_mn_major ? 1 : 0; g.b_mn = b_mn_major ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(A, lda, B, ldb, g, st);
}

int vllm_gemm_bf16_batched(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C, int ldc,
                           int n_batch, int M, int N, int K, int causal, int out_f32, void* stream) {
  // n_batch independent products C_b[M, N] = A_b . B_b^T in ONE launch: every operand / the output is a stack of its
  // n_batch matrices along the row axis (K-major A: [n_batch*M, K]; MN-major A: [n_batch*K, M]; same for B; C: [n_batch*M, N]).
  // causal (square attention matrices, M == the sequence length): see GemmArgs.  The attention-backward GEMMs of a layer.
  if (n_batch < 0 || M <= 0 || N <= 0 || K <= 0 || causal < 0 || causal > 3) return VLLM_EINVAL;
  if (causal >= 2 && K != M) return VLLM_EINVAL;     // modes 2 / 3 cut the K axis at the tile's rows: K is the sequence axis, and
                                                     // with K == M (a multiple of 256) every tile keeps at least one k-block
  if (n_batch == 0) return VLLM_OK;
  if (!A || !B || !C) return VLLM_EINVAL;
  if (M % 256 || ((a_mn_major || b_mn_major) && K % BK)) return VLLM_EUNSUPPORTED;     // tiles must not straddle matrices
  if ((long long)n_batch * M > 2147483647LL || (long long)n_batch * K > 2147483647LL || (long long)n_batch * N > 2147483647LL)
    return VLLM_EUNSUPPORTED;
  if (lda < (a_mn_major ? M : K) || ldb < (b_mn_major ? N : K) || ldc < N) return VLLM_EINVAL;
  if (!vllm_aligned(A, 16) || !vllm_aligned(B, 16) || (lda % 8) || (ldb % 8)) return VLLM_EALIGN;
  if (!vllm_aligned(C, 16) || ((size_t)ldc * (out_f32 ? 4 : 2)) % 16) return VLLM_EALIGN;
  GemmArgs g{};
  g.M = n_batch * M; g.N = N; g.K = K; g.C = C; g.ldc = ldc; g.out_f32 = out_f32;
  g.a_mn = a_mn_major ? 1 : 0; g.b_mn = b_mn_major ? 1 : 0;
  g.bt_rows = M; g.causal = causal;
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(A, lda, B, ldb, g, st);
}

int vllm_gemm_bf16_scatter(const void* A, int lda, const void* B, int ldb, void* const* dst, void* const* flags,
                           int n_dst, int rows_per_dst, int ldc, int N, int K, void* stream) {
  // C = A . B^T (plain bf16, no epilogue math), M = n_dst * rows_per_dst; row block d is stored to dst[d] and
  // counted on flags[d] (8 arrivals, one per consumer warp, per 128 x 256 tile: (rows_per_dst / 128) * ceil(N / 256) * 8 per source and pass).
  if (n_dst <= 0 || n_dst > 8 || rows_per_dst <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || ldc < N) return VLLM_EINVAL;
  if (!A || !B || !dst || !flags) return VLLM_EINVAL;
  if (rows_per_dst % BM || N % 64) return VLLM_EUNSUPPORTED;    // a tile's rows share a destination; bf16 column pairs
  if ((long long)n_dst * rows_per_dst > 2147483647LL) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(A, 16) || !vllm_aligned(B, 16) || (lda % 8) || (ldb % 8) || (ldc % 8)) return VLLM_EALIGN;
  GemmArgs g{};
  g.M = n_dst * rows_per_dst; g.N = N; g.K = K; g.ldc = ldc; g.sc_rows = rows_per_dst;
  for (int d = 0; d < n_dst; ++d) {
    if (!dst[d] || !flags[d]) return VLLM_EINVAL;
    if (!vllm_aligned(dst[d], 16)) return VLLM_EALIGN;
    g.sc_dst[d] = dst[d]; g.sc_flag[d] = (uint32_t*)flags[d];
  }
  g.C = dst[0];
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(A, lda, B, ldb, g, st);
}

int vllm_conv_rows_bf16(const void* xpad, long long pad_pixels, int channels, int padded_width, int kernel_h,
                        int kernel_w, const void* weight, int ldw, void* out, int ldo, int out_channels,
                        const void* bias, int act, void* stream) {
  // out[i, :] = epi(sum_{dy,dx} xpad[i + dy*padded_width + dx, :] . weight[:, (dy*kw + dx)*C : +C]^T) for every flat
  // pixel i of the padded map; rows whose window crosses an image edge are don't-care and sliced away by the caller.
  if (pad_pixels < 0 || channels <= 0 || padded_width <= 0 || kernel_h <= 0 || kernel_w <= 0 || out_channels <= 0)
    return VLLM_EINVAL;
  if (pad_pixels == 0) return VLLM_OK;
  if (!xpad || !weight || !out) return VLLM_EINVAL;
  if (act < 0 || act > ACT_QUICKGELU || act == ACT_SWIGLU) return VLLM_EINVAL;
  const long long seg_k = (long long)kernel_w * channels;
  // a segment must be whole k-blocks so that A's and B's K coordinates stay aligned; 16-byte row pitches
  if (seg_k % BK || channels % 8 || ldw % 8 || ldo % 8 || ldw < seg_k * kernel_h || ldo < out_channels) return VLLM_EUNSUPPORTED;
  if (pad_pixels > 2147483647LL - 4096 || seg_k * kernel_h > 2147483647LL) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(xpad, 16) || !vllm_aligned(weight, 16) || !vllm_aligned(out, 16)) return VLLM_EALIGN;
  const long long a_rows = pad_pixels - (kernel_w - 1);      // last rows whose kw-pixel span stays inside the buffer
  if (a_rows <= 0) return VLLM_EINVAL;
  GemmArgs g{};
  g.M = (int)pad_pixels; g.N = out_channels; g.K = (int)(seg_k * kernel_h); g.C = out; g.ldc = ldo;
  g.bias = (const __nv_bfloat16*)bias; g.act = act;
  g.a_seg_kb = (int)(seg_k / BK); g.a_seg_rows = padded_width;
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(xpad, channels, weight, ldw, g, st, a_rows, (int)seg_k);
}

}  // extern "C"
