// Fused attention on the sm_90a tensor cores (wgmma + TMA + mbarrier), head_dim 128 or 256.
//
// One CTA carries one 128-row Q tile of one (batch, head) and walks K/V tiles of 64 keys:
//   warpgroup 0    producer: one elected lane TMA-loads Q once and the K / V tiles into STG-deep rings (separate
//                  full / empty mbarriers for K and V, so a K stage is refilled as soon as its scores are out);
//                  the warpgroup hands its registers to the consumers.
//   warpgroups 1-2 consumers, 64 query rows each: S = Q K^T (wgmma m64n64k16, both operands from the swizzled
//                  stages) -> masks -> online softmax on the accumulator fragment (a thread holds 2 x 16 scores of two
//                  rows; row max / sum finish with two quad shuffles) -> bf16 P packed IN REGISTERS (the score fragment
//                  of two n8 blocks is the A fragment of one k16 step) -> O += P V (wgmma m64n128k16, A from registers,
//                  V MN-major from its stage).  O stays in registers (64 | 128 fp32 per thread).  The two warpgroups
//                  run unsynchronised, so one's softmax overlaps the other's MMAs.
// head_dim 256 (the GDINO bi-attention, 4 heads x 256 -- modeling_ov_grounding_dino_mask_dn.py:893-1006): Q = 4 x 16 KB
// column chunks, K/V tiles of 64 keys x 512 B, two 128-column halves of O.  KM = true adds an arbitrary key mask
// [batch, Tk] (1 = attend: the text / vision padding masks of the bi-attention); n_splits > 1 lets several CTAs share one
// query tile along the key axis (80 text queries over 21760 pixels) and write unnormalised partials in attention.cu's
// split-KV workspace layout.
#include "common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int BQ = 128, BKV = 64, THREADS = 384, CONSUMER_WARPS = 8;
template <int D> struct Cfg {
  static constexpr int NCH = D / 64;                         // 64-column (128-byte, one swizzle atom wide) chunks
  static constexpr int Q_BYTES = BQ * D * 2, Q_CHUNK = BQ * 128;
  static constexpr int KV_BYTES = BKV * D * 2, KV_CHUNK = BKV * 128;
  static constexpr int STG = D == 128 ? 4 : 2;               // 160 KB / 192 KB of Q + K/V stages
  static constexpr int SMEM = Q_BYTES + 2 * STG * KV_BYTES + 1024 + 256;
};

struct Args {
  __nv_bfloat16* o;
  long long o_bs, o_ts;
  const int* seqlens;
  int Tq, Tk, heads, kv_heads, causal;
  float scale_log2;
  const unsigned char* key_mask;   // [batch, Tk], 1 = attend (KM instantiations only)
  int n_splits;                    // CTAs per query tile along the key axis
  float* ws;                       // [batch*heads*n_splits*Tq][D + 2] fp32: unnormalised O, m (log2 domain), l
};

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));    // low half = a
  return r;
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <int D, bool KM>
__global__ void __launch_bounds__(THREADS, 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                      const __grid_constant__ CUtensorMap tm_v, const Args a) {
  constexpr int NCH = Cfg<D>::NCH, Q_BYTES = Cfg<D>::Q_BYTES, Q_CHUNK = Cfg<D>::Q_CHUNK, STG = Cfg<D>::STG;
  constexpr int KV_BYTES = Cfg<D>::KV_BYTES, KV_CHUNK = Cfg<D>::KV_CHUNK, NB = D / 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = sQ + Q_BYTES, sV = sK + STG * KV_BYTES, bar = sV + STG * KV_BYTES;
  const uint32_t q_full = bar;
  auto k_full = [&](int s) { return bar + 8 * (1 + s); };
  auto v_full = [&](int s) { return bar + 8 * (1 + STG + s); };
  auto k_empty = [&](int s) { return bar + 8 * (1 + 2 * STG + s); };
  auto v_empty = [&](int s) { return bar + 8 * (1 + 3 * STG + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x % a.n_splits;
  const int q0 = (blockIdx.x / a.n_splits) * BQ, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (a.heads / a.kv_heads);
  const int len = a.seqlens ? min(a.seqlens[b], a.Tk) : a.Tk;
  const int coff = a.Tk - a.Tq;
  int k_end = len;
  if (a.causal) k_end = min(k_end, q0 + BQ + coff);
  const int n_all = k_end > 0 ? (k_end + BKV - 1) / BKV : 0;
  const int per_split = (n_all + a.n_splits - 1) / a.n_splits;
  const int t0 = split * per_split;                        // this CTA's key tiles: [t0, t0 + n)
  const int n = max(0, min(n_all - t0, per_split));

  if (warp == 0 && lane == 0) { tc::tma_prefetch_desc(&tm_q); tc::tma_prefetch_desc(&tm_k); tc::tma_prefetch_desc(&tm_v); }
  if (warp == 1 && lane == 0) {
    tc::mbar_init(q_full, 1);
    for (int s = 0; s < STG; ++s) {
      tc::mbar_init(k_full(s), 1); tc::mbar_init(v_full(s), 1);
      tc::mbar_init(k_empty(s), CONSUMER_WARPS); tc::mbar_init(v_empty(s), CONSUMER_WARPS);
    }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    tc::reg_dealloc<40>();
    if (warp == 0 && tc::elect_one() && n > 0) {
      tc::mbar_arrive_expect_tx(q_full, Q_BYTES);
      for (int h = 0; h < NCH; ++h) tma_load_3d(sQ + h * Q_CHUNK, &tm_q, q_full, head * D + h * 64, q0, b);
      for (int j = 0; j < n; ++j) {
        const int s = j % STG;
        const uint32_t ph = ((j / STG) & 1) ^ 1;
        tc::mbar_wait(k_empty(s), ph);
        tc::mbar_arrive_expect_tx(k_full(s), KV_BYTES);
        for (int h = 0; h < NCH; ++h) tma_load_3d(sK + s * KV_BYTES + h * KV_CHUNK, &tm_k, k_full(s), kvh * D + h * 64, (t0 + j) * BKV, b);
        tc::mbar_wait(v_empty(s), ph);
        tc::mbar_arrive_expect_tx(v_full(s), KV_BYTES);
        for (int h = 0; h < NCH; ++h) tma_load_3d(sV + s * KV_BYTES + h * KV_CHUNK, &tm_v, v_full(s), kvh * D + h * 64, (t0 + j) * BKV, b);
      }
    }
    return;
  }

  // ===================== consumers: 64 query rows per warpgroup, rows r0 and r0 + 8 per thread =====================
  tc::reg_alloc<232>();
  const int wg = (warp - 4) >> 2;
  const int r0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), r1 = r0 + 8;
  const int cq = 2 * (lane & 3);                             // first column of this thread's pair inside an n8 block
  const uint32_t sQw = sQ + wg * 64 * 128;                   // this warpgroup's 64 rows of every Q chunk
  float o[NB][64];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int i = 0; i < 64; ++i) o[nb][i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // l: this thread's share of the row sums
  if (n > 0) tc::mbar_wait(q_full, 0);
  for (int j = 0; j < n; ++j) {
    const int s = j % STG;
    const uint32_t ph = (j / STG) & 1;
    // ---- S = Q K_j^T ----
    float sc[32];
    tc::mbar_wait(k_full(s), ph);
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      tc::wgmma_m64n64k16_ss(sc, tc::wgmma_desc_sw128(sQw + (kk >> 2) * Q_CHUNK + (kk & 3) * 32, 16, 1024),
                             tc::wgmma_desc_sw128(sK + s * KV_BYTES + (kk >> 2) * KV_CHUNK + (kk & 3) * 32, 16, 1024), kk != 0);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::acc_fence(sc);
    if (lane == 0) tc::mbar_arrive(k_empty(s));
    // ---- masks: sc[4*jb + 2*h + e] = (row r_h, key n0 + 8*jb + cq + e) ----
    const int n0 = (t0 + j) * BKV;
    if constexpr (KM) {
      const unsigned char* km = a.key_mask + (size_t)b * a.Tk + n0;     // the same 64 bytes for every row: cache hits
#pragma unroll
      for (int jb = 0; jb < 8; ++jb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * jb + cq + e;
          if (n0 + c < a.Tk && !__ldg(km + c)) { sc[4 * jb + e] = -INFINITY; sc[4 * jb + 2 + e] = -INFINITY; }
        }
    }
    if ((n0 + BKV > len) || (a.causal && (n0 + BKV - 1 > q0 + coff))) {
      const int lim0 = (a.causal ? min(len, r0 + coff + 1) : len) - n0;
      const int lim1 = (a.causal ? min(len, r1 + coff + 1) : len) - n0;
#pragma unroll
      for (int jb = 0; jb < 8; ++jb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * jb + cq + e;
          if (c >= lim0) sc[4 * jb + e] = -INFINITY;
          if (c >= lim1) sc[4 * jb + 2 + e] = -INFINITY;
        }
    }
    // ---- online softmax (log2 domain) ----
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int jb = 0; jb < 8; ++jb) {
      mx0 = fmaxf(mx0, fmaxf(sc[4 * jb], sc[4 * jb + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * jb + 2], sc[4 * jb + 3]));
    }
    const float mn0 = fmaxf(m0, quad_max(mx0) * a.scale_log2), mn1 = fmaxf(m1, quad_max(mx1) * a.scale_log2);
    const float corr0 = (m0 == -INFINITY) ? 0.f : ex2(m0 - mn0), corr1 = (m1 == -INFINITY) ? 0.f : ex2(m1 - mn1);
    m0 = mn0; m1 = mn1;
    const float mu0 = (m0 == -INFINITY) ? 0.f : m0, mu1 = (m1 == -INFINITY) ? 0.f : m1;   // fully masked so far: p = 0
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t p[4][4];                                        // bf16 P as the A fragments of the four k16 steps
#pragma unroll
    for (int jb = 0; jb < 8; ++jb) {
      const float p00 = ex2(fmaf(sc[4 * jb], a.scale_log2, -mu0)), p01 = ex2(fmaf(sc[4 * jb + 1], a.scale_log2, -mu0));
      const float p10 = ex2(fmaf(sc[4 * jb + 2], a.scale_log2, -mu1)), p11 = ex2(fmaf(sc[4 * jb + 3], a.scale_log2, -mu1));
      rs0 += p00 + p01; rs1 += p10 + p11;
      p[jb >> 1][(jb & 1) * 2] = pack2(p00, p01);
      p[jb >> 1][(jb & 1) * 2 + 1] = pack2(p10, p11);
    }
    l0 = l0 * corr0 + rs0; l1 = l1 * corr1 + rs1;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int i = 0; i < 64; i += 4) {
        o[nb][i] *= corr0; o[nb][i + 1] *= corr0; o[nb][i + 2] *= corr1; o[nb][i + 3] *= corr1;
      }
    // ---- O += P V_j: a k-step of 16 keys = 16 V rows x 128 B = 2 KB; columns 128.. = two 64-column chunks on ----
    tc::mbar_wait(v_full(s), ph);
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) tc::acc_fence(o[nb]);
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
        tc::wgmma_m64n128k16_rs(o[nb], p[kk], tc::wgmma_desc_sw128(sV + s * KV_BYTES + kk * 2048 + nb * 2 * KV_CHUNK, KV_CHUNK, 1024), 1);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) tc::acc_fence(o[nb]);
    if (lane == 0) tc::mbar_arrive(v_empty(s));
  }
  l0 = quad_sum(l0); l1 = quad_sum(l1);

  // ---- epilogue: column pairs (8*jb + cq, +1) of rows r0 / r1 per n8 block ----
  if (a.n_splits > 1) {
    // partial of this key range: unnormalised O, the running max (log2 domain) and the sum
    float* w0 = a.ws + ((((size_t)b * a.heads + head) * a.n_splits + split) * a.Tq + r0) * (D + 2);
    float* w1 = w0 + (size_t)8 * (D + 2);
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) {
        const int c = nb * 128 + 8 * jb + cq;
        if (r0 < a.Tq) *reinterpret_cast<float2*>(w0 + c) = make_float2(o[nb][4 * jb], o[nb][4 * jb + 1]);
        if (r1 < a.Tq) *reinterpret_cast<float2*>(w1 + c) = make_float2(o[nb][4 * jb + 2], o[nb][4 * jb + 3]);
      }
    if (cq == 0) {
      if (r0 < a.Tq) { w0[D] = m0; w0[D + 1] = l0; }
      if (r1 < a.Tq) { w1[D] = m1; w1[D + 1] = l1; }
    }
    return;
  }
  const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
  __nv_bfloat16* op0 = a.o + b * a.o_bs + (long long)r0 * a.o_ts + head * D;
  __nv_bfloat16* op1 = op0 + 8 * a.o_ts;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      const int c = nb * 128 + 8 * jb + cq;
      if (r0 < a.Tq) *reinterpret_cast<uint32_t*>(op0 + c) = pack2(o[nb][4 * jb] * inv0, o[nb][4 * jb + 1] * inv0);
      if (r1 < a.Tq) *reinterpret_cast<uint32_t*>(op1 + c) = pack2(o[nb][4 * jb + 2] * inv1, o[nb][4 * jb + 3] * inv1);
    }
}

int make_tmap(CUtensorMap* m, const void* base, uint64_t cols, uint64_t tokens, uint64_t batch, uint64_t token_pitch,
              uint64_t batch_pitch, uint32_t box_rows) {
  PFN_cuTensorMapEncodeTiled_v12000 enc = vllm_tma_encoder();
  if (!enc) return -100;
  cuuint64_t dims[3] = {cols, tokens, batch};
  cuuint64_t strides[2] = {token_pitch * 2, batch_pitch * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if (batch == 1) strides[1] = token_pitch * 2 * (tokens > 0 ? tokens : 1);
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -101;
}

}  // namespace

template <int D, bool KM>
static int launch_wgmma(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Args& a, int batch,
                        cudaStream_t st) {
  auto kern = attn_fwd_wgmma_kernel<D, KM>;
  static bool attr_set[64] = {false};
  bool* set = vllm_device_flag(attr_set);
  if (!set || !*set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<D>::SMEM);
    if (e != cudaSuccess) return (int)e;
    if (set) *set = true;
  }
  dim3 grid((unsigned)(((a.Tq + BQ - 1) / BQ) * a.n_splits), a.heads, batch);
  kern<<<grid, THREADS, Cfg<D>::SMEM, st>>>(tq, tk, tv, a);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

// head_dim 128 / 256; key_mask optional ([batch, Tk] bytes, 1 = attend); n_splits > 1: partials go to `ws`
// ([batch*heads*n_splits*Tq][head_dim + 2] fp32) and the caller merges them (attention.cu splitkv_combine_kernel).
// VLLM_EUNSUPPORTED: views a TMA descriptor cannot express (the caller then uses the warp-MMA kernel).
int vllm_attention_wgmma(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk, int heads,
                         int kv_heads, int head_dim, long long q_bs, long long q_ts, long long k_bs, long long k_ts,
                         long long v_bs, long long v_ts, long long o_bs, long long o_ts, const int* seqlens,
                         const unsigned char* key_mask, int causal, float scale, int n_splits, float* ws, cudaStream_t st) {
  if (head_dim != 128 && head_dim != 256) return VLLM_EUNSUPPORTED;
  if (n_splits < 1 || (n_splits > 1 && (!ws || causal))) return VLLM_EINVAL;
  const uint64_t D = (uint64_t)head_dim;
  CUtensorMap tq, tk, tv;
  if (make_tmap(&tq, q, (uint64_t)heads * D, Tq, batch, q_ts, q_bs, BQ)) return VLLM_EUNSUPPORTED;
  if (make_tmap(&tk, k, (uint64_t)kv_heads * D, Tk, batch, k_ts, k_bs, BKV)) return VLLM_EUNSUPPORTED;
  if (make_tmap(&tv, v, (uint64_t)kv_heads * D, Tk, batch, v_ts, v_bs, BKV)) return VLLM_EUNSUPPORTED;
  Args a;
  a.o = (__nv_bfloat16*)o; a.o_bs = o_bs; a.o_ts = o_ts; a.seqlens = seqlens; a.Tq = Tq; a.Tk = Tk;
  a.heads = heads; a.kv_heads = kv_heads; a.causal = causal; a.scale_log2 = scale * 1.4426950408889634f;
  a.key_mask = key_mask; a.n_splits = n_splits; a.ws = ws;
  if (head_dim == 128) return key_mask ? launch_wgmma<128, true>(tq, tk, tv, a, batch, st) : launch_wgmma<128, false>(tq, tk, tv, a, batch, st);
  return key_mask ? launch_wgmma<256, true>(tq, tk, tv, a, batch, st) : launch_wgmma<256, false>(tq, tk, tv, a, batch, st);
}
