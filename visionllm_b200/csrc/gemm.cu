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
//   warpgroups 1-2 consumers: warpgroup w owns rows 64(w-1)..64(w-1)+63 of the tile and issues one wgmma m64n{BN}k16
//                  per k-step straight from the swizzled stages; fp32 accumulators stay in registers
//                  (64 x BN / 128 threads = 64 | 128 per thread).  One k-block of MMAs stays in flight while the next
//                  stage is awaited; a stage goes back to the producer when the MMAs that read it have retired.
//                  The fused epilogue runs on the accumulator fragments (a thread owns column pairs of two rows, so
//                  the SwiGLU (gate, up) pair never leaves a thread).  Its operands never stall a consumer: bias,
//                  column scale and row mask of a tile come in by cp.async when the tile starts, and the first two
//                  16 x 128 B residual chunks of each warp by TMA, all under the main loop.  Each consumer warp owns
//                  two 16-row x 128-byte staging buffers (128B swizzle): the result of a chunk is written in place
//                  over its residual and leaves by one TMA store; the producer keeps prefetching the next tile meanwhile.
// Tiles are visited in groups of GROUP_M row-blocks so concurrently running CTAs share B (weights) in L2.
//
// Instantiations gemm_bf16_wgmma_kernel<BN, TA, TB, EPI> (chosen per launch by pick_kernel, 19 in all):
//   BN  128 | 256            tile width (vllm_gemm_set_variant; the scatter GEMM is always 256)
//   TA, TB  0 | 1            K-major | MN-major operand: (0, 0) for every forward call, the other three for
//                            vllm_gemm_bf16_tn / _batched / _batched_grouped (training)
//   EPI  EPI_BF16 | EPI_F32 for every (BN, TA, TB); EPI_SWIGLU for <BN, 0, 0>; EPI_SCATTER only for <256, 0, 0>
// The layout is a template parameter so that the k-block (fence, four MMAs, commit, wait) is one basic block: with a
// run-time layout branch inside it, ptxas closes the wgmma group in each branch and the wait after the join retires
// the k-block just issued.  tests/test_gemm_sass_cpu.py checks the SASS for it.
#include "common.cuh"
#include "tc_common.cuh"
#include "vllm_b200.h"   // VLLM_GEMM_* variant names

namespace {

constexpr int BM = 128, BK = 64, THREADS = 384, CONSUMER_WARPS = 8, CONSUMER_THREADS = CONSUMER_WARPS * 32;
constexpr int A_BYTES = BM * BK * 2;
constexpr int EPI_BUF = 16 * 128;                   // a staging buffer: a consumer warp's 16 rows x 128 B, 128B swizzle
constexpr int SMEM_LIMIT = 232448;                  // 227 KB: the most shared memory an sm_90 block may opt in to

enum { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2, ACT_SILU = 3, ACT_SWIGLU = 4, ACT_QUICKGELU = 5 };

struct GemmArgs {
  int M, N, K;
  void* C; int ldc;
  const __nv_bfloat16* bias; const __nv_bfloat16* colscale; const __nv_bfloat16* residual; int ldr;
  int act; int out_f32;
  const unsigned char* row_keep;   // optional [M]: rows with 0 are written as exact zeros (value.masked_fill of the MSDA module)
  int tiles_m, tiles_n;
  int group_m;           // row-blocks per rasterisation group (see launch_gemm)
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
  // Grouped batching (vllm_gemm_bf16_batched_grouped: grouped-query attention, `group` query heads per KV head).
  // reduce = 0 (broadcast): output matrix i meets A matrix i and B matrix i / group.  reduce = 1: output matrix j is the
  // sum over g < group of A_{j group + g} . B_{j group + g}^T -- both operands MN-major, so the group's K rows are
  // contiguous and the K axis is `group` segments of K rows, each with the K range of the causal mode.
  int group, reduce;
};

// Per-tile K range and operand offsets of the batched mode (identity when bt_rows == 0): the tile reads `segs` segments,
// k-blocks kb0 .. kb1 - 1 of each; segment s of an MN-major operand starts s * K rows after its k offset.
struct TilePlan { int skip, kb0, kb1, segs, b_row_off, a_k_off, b_k_off; };
__device__ __forceinline__ TilePlan plan_tile(const GemmArgs& g, int m0, int n0, int rows_per_tile, int num_kb) {
  TilePlan p{0, 0, num_kb, 1, 0, 0, 0};
  if (g.bt_rows) {
    const int bh = m0 / g.bt_rows, ml = m0 - bh * g.bt_rows;
    const int a_mat = g.reduce ? bh * g.group : bh;     // first A / B matrix the output matrix bh meets
    const int b_mat = g.reduce ? bh * g.group : bh / g.group;
    p.segs = g.reduce ? g.group : 1;
    p.b_row_off = b_mat * g.N;                          // K-major B: a stack of [N, K] matrices along the rows
    p.a_k_off = a_mat * g.K;                            // MN-major operands: stacks of [K, M|N] matrices along the K rows
    p.b_k_off = b_mat * g.K;
    if (g.causal == 1 && n0 >= ml + rows_per_tile) p.skip = 1;
    if (g.causal == 2) p.kb0 = ml / BK;
    if (g.causal == 3) { const int e = (ml + rows_per_tile + BK - 1) / BK; p.kb1 = e < num_kb ? e : num_kb; }
  }
  return p;
}

template <int BN> struct Cfg {
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // 192 KB of operand stages either way; a fifth 48 KB stage of the wide tile would need 240 KB, more than the 227 KB
  // a block may use even without the epilogue staging
  static constexpr int STAGES = BN == 256 ? 4 : 6;
  // after the stages (1024-aligned, as the 128B swizzle of the staging buffers requires): two staging buffers per
  // consumer warp, the mbarriers, then the tile's bias and column scale (bf16, BN columns + one word for a start that
  // is only 2-byte aligned) and row mask (BM bytes + one word), as cp_async_vec_word lays them out
  static constexpr int EPI_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFF = EPI_OFF + CONSUMER_WARPS * 2 * EPI_BUF;
  static constexpr int BIAS_OFF = BAR_OFF + 256;
  static constexpr int SCALE_OFF = BIAS_OFF + 2 * BN + 4;
  static constexpr int KEEP_OFF = SCALE_OFF + 2 * BN + 4;
  static constexpr int SMEM = 1024 /*align*/ + KEEP_OFF + BM + 4;
  static_assert(8 * (2 * STAGES + 2 * CONSUMER_WARPS) <= 256, "mbarriers overflow their slot");
  static_assert(SMEM <= SMEM_LIMIT, "shared memory over the per-block limit");
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

// one k-block (BK = 4 k-steps) of a warpgroup's 64 x BN tile: one m64n{BN}k16 per k-step.  B descriptor: K-major, BN
// rows of 128 B in 8-row groups 1 KB apart (SBO); MN-major, BN / 64 chunks of 64 columns 8 KB apart (LBO).
template <int BN, int TA, int TB>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint32_t sa, uint32_t sb, bool first_kb) {
  // K-major: a k-step of 16 bf16 advances the start address by 32 B inside the 128 B swizzle row;
  // MN-major: by 16 k-rows x 128 B = 2 KB (descriptor address units are 16 B)
  const uint64_t adesc = TA ? tc::wgmma_desc_sw128(sa, 8192, 1024) : tc::wgmma_desc_sw128(sa, 16, 1024);
  const uint64_t bdesc = TB ? tc::wgmma_desc_sw128(sb, 8192, 1024) : tc::wgmma_desc_sw128(sb, 16, 1024);
  constexpr uint64_t astep = TA ? 128 : 2, bstep = TB ? 128 : 2;
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    if constexpr (BN == 256)
      tc::wgmma_m64n256k16_ss<TA, TB>(acc, adesc + astep * k, bdesc + bstep * k, !(first_kb && k == 0));
    else
      tc::wgmma_m64n128k16_ss<TA, TB>(acc, adesc + astep * k, bdesc + bstep * k, !(first_kb && k == 0));
  }
}

// Epilogue of a launch (a template parameter: each instantiation carries only its own store path).  Every kind works in
// units: a unit is 16 rows x 128 B of output per consumer warp, staged in one of the warp's two buffers and stored by TMA
// (the tensor map clips the M and N tails).
//   EPI_BF16     bf16 output: a unit is 64 columns of the tile
//   EPI_SWIGLU   bf16 output of SwiGLU: a unit is 128 columns of the tile, (gate, up) pairs -> 64 output columns
//   EPI_F32      fp32 output: a unit is 64 columns of the tile, 256 B per row, so it takes both buffers
//   EPI_SCATTER  EPI_BF16 (no bias, scale, residual or mask) into the peer slots of vllm_gemm_bf16_scatter by 16-byte
//                stores from the staging buffer, then one flag arrival per consumer warp and tile
// A residual unit (64 bf16 columns, 128 B per row) is TMA-loaded into the unit's buffer (EPI_F32: buffer 0) and completes
// on that buffer's mbarrier; the thread that owns a fragment pair reads its residual and writes its result in place.
enum { EPI_BF16 = 0, EPI_SWIGLU = 1, EPI_F32 = 2, EPI_SCATTER = 3 };

// byte offset of (row r, byte b) in a 16-row x 128-byte buffer with the 128B swizzle of TMA (16-byte chunk b / 16 of
// row r sits at chunk (b / 16) ^ (r % 8); the buffer is 1024-byte aligned): the eight rows a fragment instruction touches
// (lane / 4) land in eight different bank groups
__device__ __forceinline__ int swz(int r, int b) { return r * 128 + ((((b >> 4) ^ r) & 7) << 4) + (b & 15); }

// TA / TB = 1: that operand is MN-major (vllm_gemm_bf16_tn / _batched); the layout is fixed per instantiation so that
// the k-block body is one basic block and one wgmma group stays in flight across k-blocks.
template <int BN, int TA, int TB, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r,
                       const GemmArgs g) {
  using C_ = Cfg<BN>;
  constexpr int STAGES = C_::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - tc::smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + C_::BAR_OFF;
  auto full_bar = [&](int s) { return bar_base + 8 * s; };
  auto empty_bar = [&](int s) { return bar_base + 8 * (STAGES + s); };
  auto res_bar = [&](int i) { return bar_base + 8 * (2 * STAGES + i); };   // buffer i of the staging (2 per consumer warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = g.tiles_m * g.tiles_n;
  const int num_kb = (g.K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    tc::tma_prefetch_desc(&tmap_a);
    tc::tma_prefetch_desc(&tmap_b);
    if constexpr (EPI != EPI_SCATTER) {
      tc::tma_prefetch_desc(&tmap_c);
      if (g.residual) tc::tma_prefetch_desc(&tmap_r);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), CONSUMER_WARPS); }
    for (int i = 0; i < 2 * CONSUMER_WARPS; ++i) tc::mbar_init(res_bar(i), 1);
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
        const int row_a = tm * BM - (TA ? bt_m0 : 0);
        const int row_b = tn * BN + (TB ? 0 : tp.b_row_off);
        for (int gs = 0; gs < tp.segs; ++gs) {            // grouped reduce: one segment per matrix of the group
          const int ka_off = TA ? tp.a_k_off + gs * g.K : 0, kb_off = TB ? tp.b_k_off + gs * g.K : 0;
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
            if constexpr (TA) {
              for (int h = 0; h < BM / 64; ++h) tc::tma_load_2d(sa + h * 8192, &tmap_a, full_bar(stage), ra + 64 * h, ka);
            } else {
              tc::tma_load_2d(sa, &tmap_a, full_bar(stage), ka, ra);
            }
            if constexpr (TB) {
              for (int h = 0; h < BN / 64; ++h)
                tc::tma_load_2d(sb + h * 8192, &tmap_b, full_bar(stage), row_b + 64 * h, kb * BK + kb_off);
            } else {
              tc::tma_load_2d(sb, &tmap_b, full_bar(stage), kb * BK, row_b);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: main loop + epilogue =====================
  tc::reg_alloc<232>();
  const int wg = (warp - 4) >> 2;                  // 0 / 1: rows 0-63 / 64-127 of the tile
  const int cw = warp - 4;                         // consumer warp 0..7: rows 16 cw .. 16 cw + 15 of the tile
  const int et = threadIdx.x - 128;                // 0..255
  const int lr = lane >> 2, frag_col = 2 * (lane & 3);   // fragment rows lr, lr + 8 of the warp; column pair base
  const bool has_res = EPI != EPI_SCATTER && g.residual != nullptr;
  constexpr int UNIT_COLS = EPI == EPI_SWIGLU ? 128 : 64;   // tile columns per unit
  constexpr int UNITS = BN / UNIT_COLS;
  constexpr int RES_AHEAD = EPI == EPI_F32 ? 1 : 2;         // residual units in flight (EPI_F32 stores from both buffers)
  const int n_out = EPI == EPI_SWIGLU ? g.N / 2 : g.N;
  uint8_t* s_buf = smem_gen + C_::EPI_OFF + cw * 2 * EPI_BUF;
  const uint32_t s_buf_u32 = smem_base + C_::EPI_OFF + cw * 2 * EPI_BUF;
  const uint32_t s_bias = smem_base + C_::BIAS_OFF, s_scale = smem_base + C_::SCALE_OFF, s_keep = smem_base + C_::KEEP_OFF;
  // column 0 / row 0 of a tile in those vectors: the tile starts at a multiple of 256 / 128 bytes of the global vector,
  // so its offset inside the first word is that of the vector's base
  const __nv_bfloat16* bias_t = reinterpret_cast<const __nv_bfloat16*>(smem_gen + C_::BIAS_OFF + (reinterpret_cast<uintptr_t>(g.bias) & 3));
  const __nv_bfloat16* scale_t =
      reinterpret_cast<const __nv_bfloat16*>(smem_gen + C_::SCALE_OFF + (reinterpret_cast<uintptr_t>(g.colscale) & 3));
  const uint8_t* keep_t = smem_gen + C_::KEEP_OFF + (reinterpret_cast<uintptr_t>(g.row_keep) & 3);
  // a missing bias / column scale reads as 0 / 1 for every tile: the arithmetic stays that of a present one
  if (et <= BN / 2) {
    if (!g.bias) *reinterpret_cast<uint32_t*>(smem_gen + C_::BIAS_OFF + 4 * et) = 0u;
    if (!g.colscale) *reinterpret_cast<uint32_t*>(smem_gen + C_::SCALE_OFF + 4 * et) = 0x3F803F80u;   // bf16 1.0, 1.0
  }
  uint32_t res_phase = 0;                          // bit b: parity of the next completion of buffer b's mbarrier
  int stage = 0; uint32_t phase = 0;
  float acc[BN / 2];
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    int tm, tn; tile_coords(t, g.tiles_m, g.tiles_n, g.group_m, tm, tn);
    const TilePlan tp = plan_tile(g, tm * BM, tn * BN, BM, num_kb);
    if (tp.skip) continue;
    const int n0 = tn * BN;
    const int oc0 = EPI == EPI_SWIGLU ? n0 / 2 : n0;            // the tile's first output column
    const int warp_row0 = tm * BM + cw * 16;
    const bool warp_live = warp_row0 < g.M;                     // uniform: the warp has rows to store
    // Operands of the epilogue, requested now so they arrive under the main loop.  The previous tile's readers of
    // s_bias / s_scale / s_keep left at the barrier that closed its epilogue.
    if (g.bias && et <= BN / 2) tc::cp_async_vec_word(s_bias, g.bias, 2LL * g.N, 2LL * n0, et);
    if (g.colscale && et <= BN / 2) tc::cp_async_vec_word(s_scale, g.colscale, 2LL * g.N, 2LL * n0, et);
    if (g.row_keep && et <= BM / 4) tc::cp_async_vec_word(s_keep, g.row_keep, g.M, (long long)tm * BM, et);
    auto load_res = [&](int u) {                               // lane 0: residual unit u into its buffer
      const int b = EPI == EPI_F32 ? 0 : (u & 1);
      tc::mbar_arrive_expect_tx(res_bar(2 * cw + b), EPI_BUF);
      tc::tma_load_2d(s_buf_u32 + b * EPI_BUF, &tmap_r, res_bar(2 * cw + b), oc0 + 64 * u, warp_row0);
    };
    if (has_res && warp_live && lane == 0) {
      tc::bulk_wait_read<0>();                     // the previous tile's stores have read both buffers
#pragma unroll
      for (int u = 0; u < RES_AHEAD && u < UNITS; ++u)
        if (oc0 + 64 * u < n_out) load_res(u);
    }
    int prev_stage = -1;
    const int n_kb = tp.segs * (tp.kb1 - tp.kb0);     // the producer's k-blocks of this tile, segment after segment
    for (int kb = 0; kb < n_kb; ++kb) {
      tc::mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * C_::STAGE_BYTES + wg * 8192, sb = smem_base + stage * C_::STAGE_BYTES + A_BYTES;
      const bool first = kb == 0;
      tc::acc_fence(acc);
      tc::wgmma_fence();
      mma_kblock<BN, TA, TB>(acc, sa, sb, first);
      tc::wgmma_commit();
      tc::wgmma_wait<1>();                           // the previous k-block's MMAs have retired: its stage is free
      if (prev_stage >= 0 && lane == 0) tc::mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    tc::wgmma_wait<0>();
    tc::acc_fence(acc);
    if (lane == 0) tc::mbar_arrive(empty_bar(prev_stage));
    tc::cp_async_wait_all();
    tc::named_bar_sync(1, CONSUMER_THREADS);         // every thread's cp.async of s_bias / s_scale / s_keep has landed

    // ---- epilogue on the accumulator fragments: n8 block j (columns 8j..8j+7 of the tile) is acc[4j..4j+3], the pair
    // (c, c + 1) of rows lr and lr + 8 of the warp.  Order per element: +bias -> act -> *scale -> +residual -> row mask,
    // each an fp32 operation of its own (no contraction), then one rounding to bf16.
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + frag_col;
      const float b0 = __bfloat162float(bias_t[c]), b1 = __bfloat162float(bias_t[c + 1]);
      acc[4 * j] = __fadd_rn(acc[4 * j], b0); acc[4 * j + 1] = __fadd_rn(acc[4 * j + 1], b1);
      acc[4 * j + 2] = __fadd_rn(acc[4 * j + 2], b0); acc[4 * j + 3] = __fadd_rn(acc[4 * j + 3], b1);
    }
    if constexpr (EPI == EPI_BF16 || EPI == EPI_F32) {   // one branch per tile
      switch (g.act) {
        case ACT_GELU:
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = gelu_erf(acc[i]);
          break;
        case ACT_RELU:
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = fmaxf(acc[i], 0.f);
          break;
        case ACT_SILU:
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = silu(acc[i]);
          break;
        case ACT_QUICKGELU:
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = acc[i] / (1.f + __expf(-1.702f * acc[i]));
          break;
        default: break;
      }
    }
    bool keep0 = true, keep1 = true;               // row mask of the thread's two rows
    if (g.row_keep) { keep0 = keep_t[cw * 16 + lr] != 0; keep1 = keep_t[cw * 16 + lr + 8] != 0; }

    // Output box bi of the staging (16 rows x 128 B) to columns col0.. of C.  TMA writes the columns of a row in 16-byte
    // runs, so a box that ends inside the 16-byte run holding C's last column (n_out * E not a multiple of 16) would
    // write past it: such a box -- only ever a tile's last -- goes element by element, read by the lanes before the
    // barrier that closes the tile.
    constexpr int E = EPI == EPI_F32 ? 4 : 2;
    auto put_box = [&](int bi, int col0) {
      if ((n_out * E) % 16 == 0 || col0 + 128 / E <= n_out) {
        if (lane == 0) tc::tma_store_2d(&tmap_c, s_buf_u32 + bi * EPI_BUF, col0, warp_row0);
        return;
      }
#pragma unroll
      for (int it = 0; it < 4; ++it) {               // lane: 16 bytes of row rr
        const int rr = it * 4 + (lane >> 3), piece = lane & 7, row = warp_row0 + rr;
        if (row >= g.M) continue;
#pragma unroll
        for (int e = 0; e < 16 / E; ++e) {
          const int col = col0 + piece * (16 / E) + e;
          if (col >= n_out) break;
          const uint8_t* sp = s_buf + bi * EPI_BUF + swz(rr, 16 * piece + E * e);
          uint8_t* dp = reinterpret_cast<uint8_t*>(g.C) + ((size_t)row * g.ldc + col) * E;
          if constexpr (E == 4) *reinterpret_cast<uint32_t*>(dp) = *reinterpret_cast<const uint32_t*>(sp);
          else *reinterpret_cast<uint16_t*>(dp) = *reinterpret_cast<const uint16_t*>(sp);
        }
      }
    };

    if (warp_live) {
#pragma unroll
      for (int u = 0; u < UNITS; ++u) {
        if (oc0 + 64 * u >= n_out) break;                      // uniform: the tile's last units lie past N
        const int b = EPI == EPI_F32 ? 0 : (u & 1);
        uint8_t* buf = s_buf + b * EPI_BUF;
        if (has_res) {
          // refill: the unit RES_AHEAD - 1 ahead goes to the buffer the previous unit's store has read
          if (u > 0 && u + RES_AHEAD - 1 < UNITS && oc0 + 64 * (u + RES_AHEAD - 1) < n_out && lane == 0) {
            tc::bulk_wait_read<0>();
            load_res(u + RES_AHEAD - 1);
          }
          tc::mbar_wait(res_bar(2 * cw + b), (res_phase >> b) & 1);
          res_phase ^= 1u << b;
        } else if constexpr (EPI != EPI_SCATTER && EPI != EPI_F32) {
          // the buffer's last store (two units back, or the previous tile's) has read it; the newest may still run
          if (lane == 0) { if (u == 0) tc::bulk_wait_read<0>(); else tc::bulk_wait_read<1>(); }
          __syncwarp();
        }
        if constexpr (EPI == EPI_SWIGLU) {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {                    // output column 4 jj + lane % 4 of the unit
            const int j = 16 * u + jj;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint8_t* p = buf + swz(lr + 8 * h, 16 * (jj >> 1)) + 8 * (jj & 1) + 2 * (lane & 3);
              float o = __fmul_rn(silu(acc[4 * j + 2 * h]), acc[4 * j + 2 * h + 1]);
              if (has_res) o = __fadd_rn(o, __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p)));
              *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16(o);
            }
          }
        } else {
          // *scale -> +residual -> row mask, in place in acc; EPI_BF16 / EPI_SCATTER write the pair back over its residual
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * u + jj, c = 8 * j + frag_col;
            const float s0 = __bfloat162float(scale_t[c]), s1 = __bfloat162float(scale_t[c + 1]);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float& v0 = acc[4 * j + 2 * h];
              float& v1 = acc[4 * j + 2 * h + 1];
              uint8_t* p = buf + swz(lr + 8 * h, 16 * jj) + 4 * (lane & 3);
              v0 = __fmul_rn(v0, s0); v1 = __fmul_rn(v1, s1);
              if (has_res) {
                const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
                v0 = __fadd_rn(v0, f.x); v1 = __fadd_rn(v1, f.y);
              }
              if (!(h ? keep1 : keep0)) { v0 = 0.f; v1 = 0.f; }
              if constexpr (EPI != EPI_F32) *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v0, v1);
            }
          }
          if constexpr (EPI == EPI_F32) {
            // 32 fp32 columns per buffer: every lane has read its residual from buffer 0, and both buffers' last
            // stores have read them, before any lane overwrites them
            if (lane == 0) tc::bulk_wait_read<0>();
            __syncwarp();
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * u + jj;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                uint8_t* p = s_buf + (jj >> 2) * EPI_BUF + swz(lr + 8 * h, 32 * (jj & 3) + 8 * (lane & 3));
                *reinterpret_cast<float2*>(p) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
              }
            }
          }
        }
        if constexpr (EPI == EPI_SCATTER) {
          // 16-byte stores of 128-byte row runs to the peer slot that owns row block d of C (a tile's rows share it)
          __syncwarp();
          const int d = warp_row0 / g.sc_rows;
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(g.sc_dst[d]) + (size_t)(warp_row0 - d * g.sc_rows) * g.ldc + n0 + 64 * u;
#pragma unroll
          for (int it = 0; it < 4; ++it) {             // each instruction: 4 rows x 128 contiguous bytes
            const int rr = it * 4 + (lane >> 3), piece = lane & 7;
            const uint4 val = *reinterpret_cast<const uint4*>(buf + swz(rr, 16 * piece));
            *reinterpret_cast<uint4*>(dst + (size_t)rr * g.ldc + piece * 8) = val;
          }
          __syncwarp();                                // the buffer is read before the unit two ahead rewrites it
        } else {
          // every lane's generic writes to the buffer(s) are ordered before the TMA store reads them
          tc::fence_proxy_async_smem();
          __syncwarp();
          if constexpr (EPI == EPI_F32) {
            put_box(0, n0 + 64 * u);
            if (n0 + 64 * u + 32 < n_out) put_box(1, n0 + 64 * u + 32);
          } else {
            put_box(b, oc0 + 64 * u);
          }
          if (lane == 0) tc::bulk_commit();            // one group per unit (empty when both boxes went by put_tail)
        }
      }
    }
    if constexpr (EPI == EPI_SCATTER) {                                 // tile pushed: publish it to the owner of these rows
      __threadfence_system();
      __syncwarp();
      if (lane == 0 && warp_live)
        asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(g.sc_flag[warp_row0 / g.sc_rows]), "r"(1u) : "memory");
    }
    tc::named_bar_sync(1, CONSUMER_THREADS);         // every reader of s_bias / s_scale / s_keep is done: the next tile may overwrite
  }
  // the bulk stores read shared memory and write C after their issue: both finish before the CTA exits
  if (EPI != EPI_SCATTER && lane == 0) tc::bulk_wait<0>();
}

// SM budgets (0 = every SM): a persistent GEMM CTA owns its SM (384 threads with the whole register file between them), so a
// link-bound kernel of another stream -- the peer pushes of the tensor-parallel exchange -- can only overlap a GEMM on SMs
// the GEMM's grid leaves free.  g_sm_limit caps every launch, g_scatter_sm_limit the scatter GEMM (vllm_gemm_bf16_scatter),
// whose epilogue stores ride NVLink while the other micro-batch's GEMM runs beside it (visionllm_b200/tp.py).
int g_sm_limit = 0, g_scatter_sm_limit = 0;

// VLLM_GEMM_DEFAULT: the tile width of wide_by_shape(); VLLM_GEMM_WIDE_TILE / _NARROW_TILE force the 256- / 128-column
// tile (tests and sweeps).  The scatter GEMM always uses 128 x 256: its receivers count arrivals per such tile.
int g_gemm_variant = VLLM_GEMM_DEFAULT;

using KernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const GemmArgs);

// The instantiation of a launch: operand layouts from g.a_mn / g.b_mn, epilogue from the store kind (see EPI_*).
template <int BN, int TA, int TB>
KernelFn pick_epilogue(const GemmArgs& g) {
  if (g.sc_rows) {
    if constexpr (BN == 256 && !TA && !TB) return gemm_bf16_wgmma_kernel<BN, TA, TB, EPI_SCATTER>;
    return nullptr;
  }
  if (g.act == ACT_SWIGLU) {                         // only vllm_gemm_bf16, K-major operands
    if constexpr (!TA && !TB) return gemm_bf16_wgmma_kernel<BN, TA, TB, EPI_SWIGLU>;
    return nullptr;
  }
  if (g.out_f32) return gemm_bf16_wgmma_kernel<BN, TA, TB, EPI_F32>;
  return gemm_bf16_wgmma_kernel<BN, TA, TB, EPI_BF16>;
}
template <int BN>
KernelFn pick_kernel(const GemmArgs& g) {
  if (g.a_mn) return g.b_mn ? pick_epilogue<BN, 1, 1>(g) : pick_epilogue<BN, 1, 0>(g);
  return g.b_mn ? pick_epilogue<BN, 0, 1>(g) : pick_epilogue<BN, 0, 0>(g);
}

template <int BN>
int launch_gemm(const void* A, int lda, const void* B, int ldb, GemmArgs g, cudaStream_t st, long long a_rows = -1,
                int a_cols = -1) {
  using C_ = Cfg<BN>;
  CUtensorMap ta, tb;
  // matrices in each stack (batched mode): C has nb; A has nb (broadcast) or nb * group (reduce); B has nb / group or
  // nb * group
  const uint64_t nb = g.bt_rows ? (uint64_t)(g.M / g.bt_rows) : 1;
  const uint64_t na = g.bt_rows && g.reduce ? nb * g.group : nb;
  const uint64_t nbb = !g.bt_rows ? 1 : g.reduce ? nb * g.group : nb / g.group;
  const uint64_t m_local = g.bt_rows ? (uint64_t)g.bt_rows : (uint64_t)g.M;
  int rc = g.a_mn ? vllm_make_tmap_2d(&ta, A, na * (uint64_t)g.K, m_local, (uint64_t)lda, 64)       // [K, M] rows, 64 x 64 boxes
                  : vllm_make_tmap_2d(&ta, A, (uint64_t)(a_rows < 0 ? g.M : a_rows),
                                        (uint64_t)(a_cols < 0 ? g.K : a_cols), (uint64_t)lda, BM);
  if (rc) return rc;
  rc = g.b_mn ? vllm_make_tmap_2d(&tb, B, nbb * (uint64_t)g.K, (uint64_t)g.N, (uint64_t)ldb, 64)
              : vllm_make_tmap_2d(&tb, B, nbb * (uint64_t)g.N, (uint64_t)g.K, (uint64_t)ldb, BN);
  if (rc) return rc;
  // the output and the residual in 16-row x 128-byte boxes (one staging buffer); the scatter GEMM stores to its peers directly
  CUtensorMap tc_{}, tr{};
  if (!g.sc_rows) {
    const uint64_t n_out = (uint64_t)(g.act == ACT_SWIGLU ? g.N / 2 : g.N);
    rc = vllm_make_tmap_2d(&tc_, g.C, (uint64_t)g.M, n_out, (uint64_t)g.ldc, 16, g.out_f32 != 0);
    if (!rc && g.residual) rc = vllm_make_tmap_2d(&tr, g.residual, (uint64_t)g.M, n_out, (uint64_t)g.ldr, 16);
    if (rc) return rc;
  }
  g.tiles_m = (g.M + BM - 1) / BM;
  g.tiles_n = (g.N + BN - 1) / BN;
  const int n_tiles = g.tiles_m * g.tiles_n;
  int sms = vllm_num_sms();
  const int limit = g.sc_rows ? (g_scatter_sm_limit > 0 ? g_scatter_sm_limit : g_sm_limit) : g_sm_limit;
  if (limit > 0 && limit < sms) sms = limit;
  const int ctas = sms < n_tiles ? sms : n_tiles;
  // Rasterisation: a group of `group_m` row-blocks sweeps all column-blocks before the next group starts, so one wave of
  // CTAs covers a near-square patch of tiles (minimal A+B bytes per wave).
  g.group_m = 8;
  const KernelFn kern = pick_kernel<BN>(g);
  if (!kern) return VLLM_EUNSUPPORTED;
  const cudaError_t e = vllm_smem_optin(kern, C_::SMEM);
  if (e != cudaSuccess) return (int)e;
  kern<<<ctas, THREADS, C_::SMEM, st>>>(ta, tb, tc_, tr, g);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

// Default tile width of a dense K-major GEMM: 128 x 256 when N >= 2048, else 128 x 128.  tools/gemm_bench.py, TFLOP/s
// 128 x 128 / 128 x 256 (median of 3 +- spread), each shape with its model epilogue (H100 80GB HBM3, 700 W power limit):
//   wide ahead:  LLM down 12288x4096x11008 536+-41 / 687+-8, lm_head (fp32) 12288x32026x4096 586+-9 / 648+-36,
//                gate|up (SwiGLU) 12288x22016x4096 598+-67 / 671+-7, GDINO FFN 174080x2048x256 298+-3 / 330+-4,
//                ViT qkv 41000x9600x3200 629+-15 / 673+-54
//   within the spread:  ViT proj 41000x3200x3200 620 / 613, fc1 (GELU) 41000x12800x3200 600 / 596,
//                fc2 41000x3200x12800 620 / 630, LLM qkv 12288^2x4096 684 / 692, LLM o 12288x4096x4096 581 / 570,
//                8192^3 666 / 656
// Narrower outputs, MN-major, batched and implicit-convolution launches were not measured at the wide tile and keep
// 128 x 128.
bool wide_by_shape(const GemmArgs& g) {
  return !g.a_mn && !g.b_mn && !g.bt_rows && !g.a_seg_kb && g.N >= 2048;
}

int launch_gemm_auto(const void* A, int lda, const void* B, int ldb, const GemmArgs& g, cudaStream_t st, long long a_rows = -1,
                     int a_cols = -1) {
  // the receivers of a scatter GEMM count 8 arrivals per 128 x 256 tile (visionllm_b200/tp.py)
  const bool wide = g.sc_rows || g_gemm_variant == VLLM_GEMM_WIDE_TILE ||
                    (g_gemm_variant == VLLM_GEMM_DEFAULT && wide_by_shape(g));
  return wide ? launch_gemm<256>(A, lda, B, ldb, g, st, a_rows, a_cols) : launch_gemm<128>(A, lda, B, ldb, g, st, a_rows, a_cols);
}

}  // namespace

extern "C" {

int vllm_gemm_set_variant(int v) {
  if (v != VLLM_GEMM_DEFAULT && v != VLLM_GEMM_WIDE_TILE && v != VLLM_GEMM_NARROW_TILE) return VLLM_EINVAL;
  g_gemm_variant = v;
  return VLLM_OK;
}
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

int vllm_gemm_bf16_batched_grouped(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C,
                                   int ldc, int n_batch, int group, int reduce, int M, int N, int K, int causal, int out_f32,
                                   void* stream) {
  // n_batch products A_i . B_{i / group}^T (broadcast) or n_batch / group sums of `group` products (reduce) in ONE launch;
  // every operand / the output is a stack of its matrices along the row axis (K-major A: [n*M, K]; MN-major A: [n*K, M];
  // same for B; C: [n*M, N]).  causal (square attention matrices, M == the sequence length): see GemmArgs.
  if (n_batch < 0 || M <= 0 || N <= 0 || K <= 0 || causal < 0 || causal > 3 || (reduce != 0 && reduce != 1)) return VLLM_EINVAL;
  if (group <= 0 || n_batch % group) return VLLM_EINVAL;
  if (causal >= 2 && K != M) return VLLM_EINVAL;     // modes 2 / 3 cut the K axis at the tile's rows: K is the sequence axis, and
                                                     // with K == M (a multiple of 256) every tile keeps at least one k-block
  if (reduce && (causal == 1 || causal == 3)) return VLLM_EINVAL;   // a reduce output is a key-side gradient (dK, dV)
  if (n_batch == 0) return VLLM_OK;
  if (!A || !B || !C) return VLLM_EINVAL;
  if (reduce && (!a_mn_major || !b_mn_major)) return VLLM_EUNSUPPORTED;   // the group's K rows are contiguous only MN-major
  if (M % 256 || ((a_mn_major || b_mn_major) && K % BK)) return VLLM_EUNSUPPORTED;     // tiles must not straddle matrices
  if ((long long)n_batch * M > 2147483647LL || (long long)n_batch * K > 2147483647LL || (long long)n_batch * N > 2147483647LL)
    return VLLM_EUNSUPPORTED;
  if (lda < (a_mn_major ? M : K) || ldb < (b_mn_major ? N : K) || ldc < N) return VLLM_EINVAL;
  if (!vllm_aligned(A, 16) || !vllm_aligned(B, 16) || (lda % 8) || (ldb % 8)) return VLLM_EALIGN;
  if (!vllm_aligned(C, 16) || ((size_t)ldc * (out_f32 ? 4 : 2)) % 16) return VLLM_EALIGN;
  GemmArgs g{};
  g.M = (reduce ? n_batch / group : n_batch) * M; g.N = N; g.K = K; g.C = C; g.ldc = ldc; g.out_f32 = out_f32;
  g.a_mn = a_mn_major ? 1 : 0; g.b_mn = b_mn_major ? 1 : 0;
  g.bt_rows = M; g.causal = causal; g.group = group; g.reduce = reduce;
  cudaStream_t st = (cudaStream_t)stream;
  return launch_gemm_auto(A, lda, B, ldb, g, st);
}

int vllm_gemm_bf16_batched(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C, int ldc,
                           int n_batch, int M, int N, int K, int causal, int out_f32, void* stream) {
  // n_batch independent products C_b[M, N] = A_b . B_b^T: the group = 1 broadcast of vllm_gemm_bf16_batched_grouped.
  // The attention-backward GEMMs of a layer.
  return vllm_gemm_bf16_batched_grouped(A, lda, a_mn_major, B, ldb, b_mn_major, C, ldc, n_batch, 1, 0, M, N, K, causal,
                                        out_f32, stream);
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
