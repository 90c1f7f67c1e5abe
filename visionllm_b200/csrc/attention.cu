// Fused softmax(Q K^T * scale [+ causal / length mask]) V for the ViT and LLM blocks.
//
// Replaces the reference's flash-attn 2.3.3 library calls
//   internvit/flash_attention.py:51-54 (flash_attn_varlen_qkvpacked_func, non-causal, d=128, 25 heads)
//   HF Llama FA2 / internlm2/modeling_internlm2.py:494-546 (causal, d=128, 32 heads, GQA for InternLM2)
// and the naive paths (internvit/modeling_intern_vit.py:145-160; modeling_internlm2.py:362-411).
//
// This file: FlashAttention-2 dataflow on the warp-level tensor path
// (ldmatrix + mma.sync.m16n8k16 bf16, fp32 accumulate) with online softmax in registers,
// cp.async double-buffered K/V tiles in XOR-swizzled shared memory.  CTA = 64 query rows x one head
// (4 warps x 16 rows), K/V tiles of 64 keys.  Scores never touch HBM: traffic = Q, K, V read once
// per CTA wave + O written once.  It serves head_dim 32 / 64, every attn_mask / attn_bias call and views TMA cannot
// describe; head_dim 128 / 256 otherwise run on the wgmma kernel (attention_wgmma.cu).  Attention is ~5-6 % of the
// forward FLOPs (SURVEY.md 8a-a2/a10).
//
// Layout: q/k/v are [batch, tokens, heads, D] views with arbitrary token/batch pitches (elements), so the
// packed qkv GEMM output is consumed in place; o is [batch, tokens, heads*D].  seqlens (optional, int32
// [batch]) masks keys >= len (right padding / key_padding_mask); every query row is computed (rows of
// padded queries hold finite don't-care values, as in the reference).
#include "attention.cuh"
#include "vllm_b200.h"   // VLLM_ATTN_* variant names

namespace {

constexpr int BM = 64, NW = 4;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool pred) {
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// smem tile [rows][D] bf16, 16-byte chunks XOR-swizzled with (row & 7)
template <int D>
__device__ __forceinline__ uint32_t sw_off(int row, int chunk) {
  constexpr int CH = D / 8;                       // 16-byte chunks per row
  const int x = CH >= 8 ? (row & 7) : ((row >> 1) & (CH - 1));   // D=32: two rows share a 128-byte line
  return (uint32_t)(row * D * 2 + ((chunk ^ x) << 4));
}

template <int D, int ROWS>
__device__ __forceinline__ void load_tile(uint32_t smem, const __nv_bfloat16* base, long long ts, int row0, int nrows_valid) {
  // ROWS x D tile, 128 threads, 16 B per cp.async
  constexpr int CH = D / 8;
  for (int i = threadIdx.x; i < ROWS * CH; i += NW * 32) {
    const int r = i / CH, c = i % CH;
    const bool ok = (row0 + r) < nrows_valid;
    const __nv_bfloat16* src = base + (long long)(ok ? row0 + r : 0) * ts + c * 8;
    cp_async16(smem + sw_off<D>(r, c), src, ok);
  }
}

template <int D, int BN>
__global__ void __launch_bounds__(NW * 32)
flash_fwd_kernel(const AttnArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int QB = BM * D * 2, KB = BN * D * 2;
  const uint32_t sQ = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t sK0 = sQ + QB, sV0 = sK0 + 2 * KB;

  const int split = blockIdx.x % a.n_splits, mblk = blockIdx.x / a.n_splits, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (a.heads / a.kv_heads);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int len = a.seqlens ? min(a.seqlens[b], a.Tk) : a.Tk;
  const int m0 = mblk * BM;

  const __nv_bfloat16* qb = a.q + b * a.q_bs + (long long)head * D;
  const __nv_bfloat16* kb = a.k + b * a.k_bs + (long long)kvh * D;
  const __nv_bfloat16* vb = a.v + b * a.v_bs + (long long)kvh * D;
  __nv_bfloat16* ob = a.o + b * a.o_bs + (long long)head * D;

  // causal offset: query i attends keys <= i + (Tk - Tq)  (bottom-right aligned, like flash-attn)
  const int coff = a.Tk - a.Tq;
  int k_end = len;
  if (a.causal) k_end = min(k_end, m0 + BM + coff);
  const int n_tiles_all = (k_end + BN - 1) / BN;
  // split-KV: this CTA owns key tiles [t_begin, t_begin + n_tiles)
  const int per_split = (n_tiles_all + a.n_splits - 1) / a.n_splits;
  const int t_begin = split * per_split;
  int n_tiles = max(0, min(n_tiles_all, t_begin + per_split) - t_begin);
  const int* live = nullptr;                                    // live-tile list of this (batch, head, query block)
  if (BN == 64 && a.tile_counts) {
    const long long item = ((long long)b * a.heads + head) * a.q_blocks + mblk;
    n_tiles = a.tile_counts[item];
    live = a.tile_lists + item * a.k_tiles;
  }
  auto tile_id = [&](int t) { return live ? live[t] : t_begin + t; };

  load_tile<D, BM>(sQ, qb, a.q_ts, m0, a.Tq);
  cp_async_commit();
  if (n_tiles > 0) {
    load_tile<D, BN>(sK0, kb, a.k_ts, tile_id(0) * BN, len);
    load_tile<D, BN>(sV0, vb, a.v_ts, tile_id(0) * BN, len);
  }
  cp_async_commit();

  // Q fragments -> registers
  cp_async_wait<1>();
  __syncthreads();
  uint32_t qf[D / 16][4];
  {
    const int r = warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const int chunk = kk * 2 + (lane >> 4);
      ldsm_x4(sQ + sw_off<D>(r, chunk), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
    }
  }

  float o[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const int g = lane >> 2, tq = lane & 3;
  const int qrow0 = m0 + warp * 16 + g;  // and +8

  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t & 1;
    const uint32_t sK = sK0 + buf * KB, sV = sV0 + buf * KB;
    if (t + 1 < n_tiles) {
      load_tile<D, BN>(sK0 + (buf ^ 1) * KB, kb, a.k_ts, tile_id(t + 1) * BN, len);
      load_tile<D, BN>(sV0 + (buf ^ 1) * KB, vb, a.v_ts, tile_id(t + 1) * BN, len);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[BN / 8][4];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int j = 0; j < BN / 8; j += 2) {
        const int key = j * 8 + (lane & 7) + 8 * (lane >> 4);
        const int chunk = kk * 2 + ((lane >> 3) & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(sK + sw_off<D>(key, chunk), b0, b1, b2, b3);
        mma_bf16(s[j], qf[kk], b0, b1);
        mma_bf16(s[j + 1], qf[kk], b2, b3);
      }
    }
    // ---- mask + online softmax (scores scaled into log2 domain) ----
    const int n0 = tile_id(t) * BN;
    const unsigned char* km = a.key_mask ? a.key_mask + (long long)b * a.Tk : nullptr;
    const unsigned char* am = a.attn_mask ? a.attn_mask + ((long long)b * a.heads + head) * a.Tq * a.Tk : nullptr;
    const float* ab = a.attn_bias
                          ? a.attn_bias + ((long long)(b % a.bias_batches) * a.heads + head) * a.Tq * a.Tk : nullptr;
    const bool need_mask = km || am || ab || (n0 + BN > len) || (a.causal && (n0 + BN - 1 > m0 + coff));
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s[j][e] * a.scale_log2;
        if (need_mask) {
          const int key = n0 + j * 8 + tq * 2 + (e & 1);
          const int qr = qrow0 + (e >> 1) * 8;
          if (key >= len || (a.causal && key > qr + coff) || (km && !km[key]) ||
              (am && qr < a.Tq && !am[(long long)qr * a.Tk + key]))
            v = -INFINITY;
          else if (ab && qr < a.Tq)
            v = fmaf(ab[(long long)qr * a.Tk + key], 1.4426950408889634f, v);
        }
        s[j][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mnew = fmaxf(mrow[r], mx[r]);
      const float msafe = (mnew == -INFINITY) ? 0.f : mnew;
      corr[r] = exp2f(mrow[r] - msafe);   // mrow = -inf -> 0
      mrow[r] = mnew;
      mx[r] = msafe;
      lrow[r] *= corr[r];
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = exp2f(s[j][e] - mx[e >> 1]);
        s[j][e] = p;
        rs[e >> 1] += p;
      }
    }
    lrow[0] += rs[0]; lrow[1] += rs[1];
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1];
    }
    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      uint32_t pa[4];
      pa[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int j = 0; j < D / 8; j += 2) {
        const int key = kk * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
        const int chunk = j + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(sV + sw_off<D>(key, chunk), b0, b1, b2, b3);
        mma_bf16(o[j], pa, b0, b1);
        mma_bf16(o[j + 1], pa, b2, b3);
      }
    }
    __syncthreads();  // tile buffers are overwritten by the next iteration's prefetch
  }

  // ---- finalize: O / l, write bf16 ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
  }
  if (a.n_splits > 1) {
    // partial result of this key range: unnormalised O, running max (log2 domain) and sum
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = qrow0 + r * 8;
      if (row >= a.Tq) continue;
      float* wp = a.ws + ((((size_t)b * a.heads + head) * a.n_splits + split) * a.Tq + row) * (D + 2);
#pragma unroll
      for (int j = 0; j < D / 8; ++j)
        *reinterpret_cast<float2*>(wp + j * 8 + tq * 2) = make_float2(o[j][2 * r], o[j][2 * r + 1]);
      if (tq == 0) { wp[D] = mrow[r]; wp[D + 1] = lrow[r]; }
    }
    return;
  }
  const float inv0 = lrow[0] > 0.f ? 1.f / lrow[0] : 0.f, inv1 = lrow[1] > 0.f ? 1.f / lrow[1] : 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = qrow0 + r * 8;
    if (row >= a.Tq) continue;
    const bool live = true;
    __nv_bfloat16* op = ob + (long long)row * a.o_ts;
    const float inv = r ? inv1 : inv0;
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const float x = live ? o[j][2 * r] * inv : 0.f, y = live ? o[j][2 * r + 1] * inv : 0.f;
      *reinterpret_cast<__nv_bfloat162*>(op + j * 8 + tq * 2) = __floats2bfloat162_rn(x, y);
    }
  }
}

// Live-tile lists of an attn_mask [n_bh, Tq, Tk] (1 = attend): one CTA per (bh, 64-row query block) walks the 64-key tiles,
// ORs the 64 x 64 bytes of each block-wide and appends the ids of the non-empty ones.
__global__ void __launch_bounds__(256)
mask_tiles_kernel(const unsigned char* __restrict__ mask, int Tq, int Tk, int q_blocks, int k_tiles, int* __restrict__ counts,
                  int* __restrict__ lists) {
  const long long item = blockIdx.x;                            // bh * q_blocks + qb
  const int qb = (int)(item % q_blocks);
  const long long bh = item / q_blocks;
  const unsigned char* m = mask + bh * (long long)Tq * Tk;
  const int r = threadIdx.x >> 2, c0 = (threadIdx.x & 3) * 16;  // thread: row r of the block, 16 consecutive keys
  const int row = qb * 64 + r;
  int n = 0;
  for (int kt = 0; kt < k_tiles; ++kt) {
    int any = 0;
    if (row < Tq) {
      const unsigned char* p = m + (long long)row * Tk + kt * 64 + c0;
#pragma unroll
      for (int j = 0; j < 16; ++j) any |= (kt * 64 + c0 + j < Tk) ? p[j] : 0;
    }
    if (__syncthreads_or(any)) {
      if (threadIdx.x == 0) lists[item * k_tiles + n] = kt;
      ++n;
    }
  }
  if (threadIdx.x == 0) counts[item] = n;
}

// merge the split-KV partials of one query row: one warp per (batch, head, row), lanes over head_dim
template <int D>
__global__ void __launch_bounds__(128)
splitkv_combine_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ o, long long o_bs, long long o_ts,
                       int Tq, int heads, int n_splits, long long n_rows) {
  const long long wid = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const int row = (int)(wid % Tq);
  const long long bh = wid / Tq;
  const int head = (int)(bh % heads);
  const long long b = bh / heads;
  float m = -INFINITY;
  for (int s = 0; s < n_splits; ++s) m = fmaxf(m, ws[((bh * n_splits + s) * Tq + row) * (D + 2) + D]);
  const float msafe = (m == -INFINITY) ? 0.f : m;
  float l = 0.f;
  float acc[D / 32];
#pragma unroll
  for (int i = 0; i < D / 32; ++i) acc[i] = 0.f;
  for (int s = 0; s < n_splits; ++s) {
    const float* wp = ws + ((bh * n_splits + s) * Tq + row) * (D + 2);
    const float sc = exp2f(wp[D] - msafe);      // -inf -> 0 for empty ranges
    l += wp[D + 1] * sc;
#pragma unroll
    for (int i = 0; i < D / 32; ++i) acc[i] += wp[lane + 32 * i] * sc;
  }
  const float inv = l > 0.f ? 1.f / l : 0.f;
  __nv_bfloat16* op = o + b * o_bs + (long long)row * o_ts + (long long)head * D;
#pragma unroll
  for (int i = 0; i < D / 32; ++i) op[lane + 32 * i] = __float2bfloat16(acc[i] * inv);
}

// ---------------------------------------------------------------------------------------------------------------------
// Window attention (Swin: head_dim 32, <= 64 tokens per window, additive fp32 bias slab = relative-position bias +
// shifted-window mask, HF SwinSelfAttention / modeling_unipose.py:1277-1354): ONE WARP per (window, head), four independent
// warps per CTA walking a strided item list -- no block-wide barrier anywhere, so 16 resident warps per SM overlap their
// global-load latencies (the general kernel above spends a whole CTA and three __syncthreads on one 49 x 49 problem:
// 33 k CTAs per Swin-T stage-1 layer at 1024^2).  Per item the warp stages Q / K / V (<= 64 rows x 64 B each) in its own
// 12 KB of shared memory with cp.async, then for each 16-row query tile: bias loads issued first, S = Q K^T (16 HMMA),
// softmax in registers, O = P V (16 HMMA), one 64-byte store per row.  Same arithmetic order as flash_fwd_kernel<32, 64>
// for a single key tile (scores in the log2 domain, fp32 softmax, bf16 P), so results are bit-identical to it.
// ---------------------------------------------------------------------------------------------------------------------
struct WinArgs {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* o;
  long long q_bs, k_bs, v_bs, o_bs, q_ts, k_ts, v_ts, o_ts;
  const float* bias;               // [bias_batches, heads, T, T]
  int bias_batches, T, heads;
  long long n_items;               // batch (= windows) x heads
  float scale_log2;
};

__global__ void __launch_bounds__(128, 4)
window_attn_kernel(const WinArgs a) {
  constexpr int D = 32, ROWS = 64, CH = D / 8, TILE = ROWS * D * 2;
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sQ = (uint32_t)__cvta_generic_to_shared(smem) + warp * 3 * TILE, sK = sQ + TILE, sV = sK + TILE;
  const int g = lane >> 2, tq = lane & 3;
  const int T = a.T;
  for (long long item = (long long)blockIdx.x * 4 + warp; item < a.n_items; item += (long long)gridDim.x * 4) {
    const long long b = item / a.heads;
    const int head = (int)(item - b * a.heads);
    const __nv_bfloat16* qb = a.q + b * a.q_bs + (long long)head * D;
    const __nv_bfloat16* kb = a.k + b * a.k_bs + (long long)head * D;
    const __nv_bfloat16* vb = a.v + b * a.v_bs + (long long)head * D;
    __syncwarp();                                          // the previous item's ldmatrix reads are done
    for (int i = lane; i < ROWS * CH; i += 32) {
      const int r = i / CH, c = i % CH;
      const bool ok = r < T;
      const long long rr = ok ? r : 0;
      cp_async16(sQ + sw_off<D>(r, c), qb + rr * a.q_ts + c * 8, ok);
      cp_async16(sK + sw_off<D>(r, c), kb + rr * a.k_ts + c * 8, ok);
      cp_async16(sV + sw_off<D>(r, c), vb + rr * a.v_ts + c * 8, ok);
    }
    cp_async_commit();
    const float* ab = a.bias + (((long long)(b % a.bias_batches)) * a.heads + head) * T * T;
    cp_async_wait<0>();
    __syncwarp();
    __nv_bfloat16* ob = a.o + b * a.o_bs + (long long)head * D;
    const int n_mt = (T + 15) / 16;
    for (int mt = 0; mt < n_mt; ++mt) {
      // bias of this thread's score fragment first: the loads fly while the Q / K fragments are fetched and multiplied
      const int qr0 = mt * 16 + g;
      float bv[ROWS / 8][4];
#pragma unroll
      for (int j = 0; j < ROWS / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = j * 8 + tq * 2 + (e & 1), qr = qr0 + (e >> 1) * 8;
          bv[j][e] = (key < T && qr < T) ? __ldg(ab + (long long)qr * T + key) : 0.f;
        }
      uint32_t qf[D / 16][4];
      {
        const int r = mt * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
          const int chunk = kk * 2 + (lane >> 4);
          ldsm_x4(sQ + sw_off<D>(r, chunk), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
        }
      }
      float s[ROWS / 8][4];
#pragma unroll
      for (int j = 0; j < ROWS / 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
        for (int j = 0; j < ROWS / 8; j += 2) {
          const int key = j * 8 + (lane & 7) + 8 * (lane >> 4);
          const int chunk = kk * 2 + ((lane >> 3) & 1);
          uint32_t b0, b1, b2, b3;
          ldsm_x4(sK + sw_off<D>(key, chunk), b0, b1, b2, b3);
          mma_bf16(s[j], qf[kk], b0, b1);
          mma_bf16(s[j + 1], qf[kk], b2, b3);
        }
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < ROWS / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = j * 8 + tq * 2 + (e & 1), qr = qr0 + (e >> 1) * 8;
          float v = s[j][e] * a.scale_log2;
          if (key >= T) v = -INFINITY;
          else if (qr < T) v = fmaf(bv[j][e], 1.4426950408889634f, v);
          s[j][e] = v;
          mx[e >> 1] = fmaxf(mx[e >> 1], v);
        }
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        if (mx[r] == -INFINITY) mx[r] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < ROWS / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = exp2f(s[j][e] - mx[e >> 1]);
          s[j][e] = p;
          rs[e >> 1] += p;
        }
      }
      float o[D / 8][4];
#pragma unroll
      for (int j = 0; j < D / 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < ROWS / 16; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
        pa[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
        pa[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pa[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
        for (int j = 0; j < D / 8; j += 2) {
          const int key = kk * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
          const int chunk = j + (lane >> 4);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(sV + sw_off<D>(key, chunk), b0, b1, b2, b3);
          mma_bf16(o[j], pa, b0, b1);
          mma_bf16(o[j + 1], pa, b2, b3);
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
        const int row = qr0 + r * 8;
        if (row < T) {
          const float inv = rs[r] > 0.f ? 1.f / rs[r] : 0.f;
          __nv_bfloat16* op = ob + (long long)row * a.o_ts;
#pragma unroll
          for (int j = 0; j < D / 8; ++j)
            *reinterpret_cast<__nv_bfloat162*>(op + j * 8 + tq * 2) = __floats2bfloat162_rn(o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
        }
      }
    }
  }
}

static int launch_window(const AttnArgs& a, int batch, cudaStream_t st) {
  constexpr int SMEM = 4 * 3 * 64 * 32 * 2;               // 4 warps x (Q, K, V) x 64 rows x 64 B
  const cudaError_t e = vllm_smem_optin(window_attn_kernel, SMEM);
  if (e != cudaSuccess) return (int)e;
  WinArgs w;
  w.q = a.q; w.k = a.k; w.v = a.v; w.o = a.o;
  w.q_bs = a.q_bs; w.k_bs = a.k_bs; w.v_bs = a.v_bs; w.o_bs = a.o_bs;
  w.q_ts = a.q_ts; w.k_ts = a.k_ts; w.v_ts = a.v_ts; w.o_ts = a.o_ts;
  w.bias = a.attn_bias; w.bias_batches = a.bias_batches; w.T = a.Tq; w.heads = a.heads;
  w.n_items = (long long)batch * a.heads; w.scale_log2 = a.scale_log2;
  long long ctas = (w.n_items + 3) / 4;
  const long long cap = (long long)vllm_num_sms() * 4 * 4;  // 4 resident CTAs per SM, a few items per warp
  if (ctas > cap) ctas = cap;
  window_attn_kernel<<<(unsigned)ctas, 128, SMEM, st>>>(w);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

// Split-KV: when the query tiles alone cannot fill the GPU (e.g. 80 text queries over 21760 pixels), several CTAs share one
// query tile along the key axis, write unnormalised partials to the workspace, and splitkv_combine_kernel merges them.
// The constants of one kernel family:
struct SplitKv {
  int q_tile, k_tile;   // query rows / keys per tile
  int per_sm;           // resident CTAs per SM
  int tiles_per_split;  // largest split count = min(key tiles / tiles_per_split, 64)
  int fixed_tiles;      // fixed cost of a CTA (Q load, prologue, partial write-out) in key tiles
  bool reject_empty;    // skip counts that would leave the last split(s) without a key tile
};

// The split count (1 = none) that minimises (waves of resident CTAs) x (key tiles per split + fixed cost): a count that
// spills a few CTAs into one more wave costs a whole extra pass.  The partials of a count must fit the workspace.
static int split_kv_count(const AttnArgs& a, int batch, int D, const SplitKv& f, const void* workspace,
                          long long workspace_bytes) {
  const long long ctas = (long long)((a.Tq + f.q_tile - 1) / f.q_tile) * a.heads * batch;
  const int n_tiles = (a.Tk + f.k_tile - 1) / f.k_tile;
  if (!workspace || a.causal || a.tile_counts || ctas >= 2LL * vllm_num_sms() || n_tiles < 16) return 1;
  const long long slots = (long long)vllm_num_sms() * f.per_sm;
  long long best = 1, best_cost = (ctas + slots - 1) / slots * (n_tiles + f.fixed_tiles);
  const long long max_s = n_tiles / f.tiles_per_split < 64 ? n_tiles / f.tiles_per_split : 64;
  for (long long sp = 2; sp <= max_s; ++sp) {
    if ((long long)batch * a.heads * sp * a.Tq * (D + 2) * 4 > workspace_bytes) break;
    if (f.reject_empty && (sp - 1) * ((n_tiles + sp - 1) / sp) >= n_tiles) continue;
    const long long waves = (ctas * sp + slots - 1) / slots;
    const long long cost = waves * ((n_tiles + sp - 1) / sp + f.fixed_tiles);
    if (cost < best_cost) { best_cost = cost; best = sp; }
  }
  return (int)best;
}

int g_attn_splits = 0;  // vllm_attention_set_splits: 0 = split_kv_count decides, 1..64 = that count

// The split count of a call: the count forced by vllm_attention_set_splits, else split_kv_count's.  VLLM_EINVAL when the
// workspace cannot hold the forced count's partials.  A NULL workspace and a tile-list call never split.
static int splits_of(const AttnArgs& a, int batch, int D, const SplitKv& f, const void* workspace, long long workspace_bytes) {
  if (!g_attn_splits) return split_kv_count(a, batch, D, f, workspace, workspace_bytes);
  if (!workspace || a.tile_counts) return 1;
  if ((long long)batch * a.heads * g_attn_splits * a.Tq * (D + 2) * 4 > workspace_bytes) return VLLM_EINVAL;
  return g_attn_splits;
}

template <int D>
static int launch_combine(const AttnArgs& a, int batch, cudaStream_t st) {
  const long long n_rows = (long long)batch * a.heads * a.Tq;
  splitkv_combine_kernel<D><<<(unsigned)((n_rows + 3) / 4), 128, 0, st>>>(a.ws, a.o, a.o_bs, a.o_ts, a.Tq, a.heads,
                                                                         a.n_splits, n_rows);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

template <int D, int BN = 64>
int launch(AttnArgs a, int batch, cudaStream_t st, void* workspace, long long workspace_bytes) {
  constexpr int SMEM = BM * D * 2 + 4 * BN * D * 2;
  const cudaError_t e = vllm_smem_optin(flash_fwd_kernel<D, BN>, SMEM);
  if (e != cudaSuccess) return (int)e;
  static int per_sm = 0;                                  // depends on the kernel and the architecture only
  if (!per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flash_fwd_kernel<D, BN>, NW * 32, SMEM) != cudaSuccess ||
                  per_sm < 1))
    per_sm = 1;
  a.n_splits = splits_of(a, batch, D, {BM, BN, per_sm, 8, 2, false}, workspace, workspace_bytes);
  if (a.n_splits < 1) return a.n_splits;
  a.ws = a.n_splits > 1 ? (float*)workspace : nullptr;
  dim3 grid((unsigned)(((a.Tq + BM - 1) / BM) * a.n_splits), a.heads, batch);
  flash_fwd_kernel<D, BN><<<grid, NW * 32, SMEM, st>>>(a);
  VLLM_CHECK_LAUNCH();
  return a.n_splits > 1 ? launch_combine<D>(a, batch, st) : VLLM_OK;
}

// The wgmma kernel (attention_wgmma.cu) runs one CTA of 128 query rows per SM.  An unmasked head_dim-128 call never
// splits, and only this family rejects empty splits: both as tuned so far (the split-KV re-tune, DESIGN §10 item 3).
// A count forced by vllm_attention_set_splits overrides both.
template <int D>
static int launch_wgmma(AttnArgs a, int batch, cudaStream_t st, void* workspace, long long workspace_bytes) {
  if (D == 128 && !a.key_mask && !g_attn_splits) workspace = nullptr;
  a.n_splits = splits_of(a, batch, D, {128, 64, 1, 4, 4, true}, workspace, workspace_bytes);
  if (a.n_splits < 1) return a.n_splits;
  a.ws = a.n_splits > 1 ? (float*)workspace : nullptr;
  const int rc = vllm_attention_wgmma(a, batch, D, st);
  return rc == VLLM_OK && a.n_splits > 1 ? launch_combine<D>(a, batch, st) : rc;
}

}  // namespace

static int g_attn_variant = VLLM_ATTN_DEFAULT;  // see vllm_attention_set_variant
extern "C" int vllm_attention_set_variant(int v) {
  if (v != VLLM_ATTN_DEFAULT && v != VLLM_ATTN_WARP_MMA) return VLLM_EINVAL;
  g_attn_variant = v;
  return VLLM_OK;
}
extern "C" int vllm_attention_set_splits(int n) {
  if (n < 0 || n > 64) return VLLM_EINVAL;
  g_attn_splits = n;
  return VLLM_OK;
}

static int attention_impl(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk,
                          int heads, int kv_heads, int head_dim, long long q_batch_pitch,
                          long long q_token_pitch, long long k_batch_pitch, long long k_token_pitch,
                          long long v_batch_pitch, long long v_token_pitch, long long o_batch_pitch,
                          long long o_token_pitch, const int* seqlens, const unsigned char* key_mask,
                          const unsigned char* attn_mask, const float* attn_bias, int bias_batches,
                          int causal, float scale, void* workspace, long long workspace_bytes, const int* tile_counts,
                          const int* tile_lists, void* stream) {
  if (batch < 0 || Tq < 0 || Tk < 0 || heads <= 0 || kv_heads <= 0 || heads % kv_heads) return VLLM_EINVAL;
  // The wgmma kernel takes the row max of the unscaled scores: a scale <= 0 would turn the masked -inf into +inf / NaN.
  if (!(scale > 0.f) || !isfinite(scale)) return VLLM_EINVAL;
  if ((tile_counts == nullptr) != (tile_lists == nullptr)) return VLLM_EINVAL;
  if (tile_counts && (!attn_mask || causal || (head_dim != 32 && head_dim != 64 && head_dim != 128))) return VLLM_EUNSUPPORTED;
  if (batch == 0 || Tq == 0) return VLLM_OK;
  if (!q || !k || !v || !o) return VLLM_EINVAL;
  if (attn_bias && bias_batches <= 0) return VLLM_EINVAL;
  if (batch > 65535 || heads > 65535) return VLLM_EUNSUPPORTED;
  const long long p[] = {q_batch_pitch, q_token_pitch, k_batch_pitch, k_token_pitch,
                         v_batch_pitch, v_token_pitch, o_batch_pitch, o_token_pitch};
  for (long long x : p) if (x % 8) return VLLM_EALIGN;
  if (!vllm_aligned(q, 16) || !vllm_aligned(k, 16) || !vllm_aligned(v, 16) || !vllm_aligned(o, 16)) return VLLM_EALIGN;
  AttnArgs a;
  a.q = (const __nv_bfloat16*)q; a.k = (const __nv_bfloat16*)k; a.v = (const __nv_bfloat16*)v;
  a.o = (__nv_bfloat16*)o;
  a.q_bs = q_batch_pitch; a.k_bs = k_batch_pitch; a.v_bs = v_batch_pitch; a.o_bs = o_batch_pitch;
  a.q_ts = q_token_pitch; a.k_ts = k_token_pitch; a.v_ts = v_token_pitch; a.o_ts = o_token_pitch;
  a.seqlens = seqlens; a.key_mask = key_mask; a.attn_mask = attn_mask; a.attn_bias = attn_bias; a.bias_batches = bias_batches; a.Tq = Tq; a.Tk = Tk; a.heads = heads; a.kv_heads = kv_heads; a.causal = causal;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.n_splits = 1; a.ws = nullptr;
  a.tile_counts = tile_counts; a.tile_lists = tile_lists; a.q_blocks = (Tq + 63) / 64; a.k_tiles = (Tk + 63) / 64;
  cudaStream_t st = (cudaStream_t)stream;
  // The first kernel that takes the call runs it; VLLM_ATTN_WARP_MMA leaves only the last one.
  const bool all_kernels = g_attn_variant == VLLM_ATTN_DEFAULT;
  // 1. wgmma: head_dim 128 / 256 without attn_mask / attn_bias; a view a TMA descriptor cannot express goes on to 3.
  if (all_kernels && (head_dim == 128 || head_dim == 256) && !attn_mask && !attn_bias) {
    const int rc = head_dim == 128 ? launch_wgmma<128>(a, batch, st, workspace, workspace_bytes)
                                   : launch_wgmma<256>(a, batch, st, workspace, workspace_bytes);
    if (rc != VLLM_EUNSUPPORTED) return rc;
  }
  // 2. Swin windows: head_dim 32, one key tile, additive bias only -> one warp per (window, head)
  if (all_kernels && head_dim == 32 && attn_bias && !key_mask && !attn_mask && !seqlens && !causal && Tq == Tk && Tq <= 64 &&
      kv_heads == heads)
    return launch_window(a, batch, st);
  // 3. the warp-MMA kernel
  switch (head_dim) {
    case 128: return launch<128>(a, batch, st, workspace, workspace_bytes);
    case 64: return launch<64>(a, batch, st, workspace, workspace_bytes);
    case 32: return launch<32>(a, batch, st, workspace, workspace_bytes);
    case 256: return launch<256, 32>(a, batch, st, workspace, workspace_bytes);
    default: return VLLM_EUNSUPPORTED;
  }
}

extern "C" int vllm_attention_bf16(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk,
                                   int heads, int kv_heads, int head_dim, long long q_batch_pitch,
                                   long long q_token_pitch, long long k_batch_pitch, long long k_token_pitch,
                                   long long v_batch_pitch, long long v_token_pitch, long long o_batch_pitch,
                                   long long o_token_pitch, const int* seqlens, const unsigned char* key_mask,
                                   const unsigned char* attn_mask, const float* attn_bias, int bias_batches,
                                   int causal, float scale, void* workspace, long long workspace_bytes, void* stream) {
  return attention_impl(q, k, v, o, batch, Tq, Tk, heads, kv_heads, head_dim, q_batch_pitch, q_token_pitch, k_batch_pitch,
                        k_token_pitch, v_batch_pitch, v_token_pitch, o_batch_pitch, o_token_pitch, seqlens, key_mask, attn_mask,
                        attn_bias, bias_batches, causal, scale, workspace, workspace_bytes, nullptr, nullptr, stream);
}

extern "C" int vllm_attention_bf16_tiles(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk,
                                         int heads, int kv_heads, int head_dim, long long q_batch_pitch,
                                         long long q_token_pitch, long long k_batch_pitch, long long k_token_pitch,
                                         long long v_batch_pitch, long long v_token_pitch, long long o_batch_pitch,
                                         long long o_token_pitch, const int* seqlens, const unsigned char* key_mask,
                                         const unsigned char* attn_mask, float scale, const int* tile_counts,
                                         const int* tile_lists, void* stream) {
  if (!tile_counts || !tile_lists) return VLLM_EINVAL;
  return attention_impl(q, k, v, o, batch, Tq, Tk, heads, kv_heads, head_dim, q_batch_pitch, q_token_pitch, k_batch_pitch,
                        k_token_pitch, v_batch_pitch, v_token_pitch, o_batch_pitch, o_token_pitch, seqlens, key_mask, attn_mask,
                        nullptr, 0, 0, scale, nullptr, 0, tile_counts, tile_lists, stream);
}

extern "C" int vllm_attention_mask_tiles(const unsigned char* attn_mask, long long n_batch_heads, int Tq, int Tk, int* tile_counts,
                                         int* tile_lists, void* stream) {
  if (n_batch_heads < 0 || Tq < 0 || Tk < 0) return VLLM_EINVAL;
  if (n_batch_heads == 0 || Tq == 0) return VLLM_OK;
  if (!attn_mask || !tile_counts || !tile_lists) return VLLM_EINVAL;
  const int q_blocks = (Tq + 63) / 64, k_tiles = (Tk + 63) / 64;
  const long long items = n_batch_heads * q_blocks;
  if (items > 2147483647LL) return VLLM_EUNSUPPORTED;
  mask_tiles_kernel<<<(unsigned)items, 256, 0, (cudaStream_t)stream>>>(attn_mask, Tq, Tk, q_blocks, k_tiles, tile_counts, tile_lists);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}
