// Multi-scale deformable attention (MSDA) forward for sm_90a.
//
// Replaces the reference operator
//   mmcv/ops/csrc/common/cuda/ms_deform_attn_cuda_kernel.cuh:17-64,200-254
//   (== visionllmv2/model/unipose/ops/src/cuda/ms_deform_im2col_cuda.cuh:33-85,237-300)
// behind the C-ABI declared in include/vllm_b200.h.
//
// Data layout (all contiguous, identical to the reference extension):
//   value  [N, S, M, D]          S = sum_l H_l*W_l, level-major, row-major
//   shapes [L, 2] int64 (H, W)   on the DEVICE, like the reference
//   lsi    [L]    int64          level start index, on the DEVICE
//   loc    [N, Lq, M, L, P, 2]   (x, y) normalised
//   attw   [N, Lq, M, L, P]
//   out    [N, Lq, M*D]
//
// Two kernels:
//  * msda_fwd_strict_kernel<T>: one thread per output scalar, the reference's
//    arithmetic and summation order with every product/sum individually
//    rounded (no FMA contraction).  Any D / L / P, fp32 and fp64.  Bit-exact
//    against oracle/msda_oracle.c.
//  * msda_fwd_warp_kernel: the fast fp32 path for D == 32.  One warp owns a
//    (query, head) pair.  Phase 1: one lane per (level, point) sample does the
//    index arithmetic ONCE (the reference repeats it in all D threads) and
//    writes {element offset, bilinear*attention weight} per corner to a
//    warp-private shared-memory slab.  Phase 2: lane = (corner, channel quad):
//    one predicated LDG.128 per lane fetches the four 128-byte corner rows of
//    a sample in a single instruction; each lane FMAs into a float4
//    accumulator; two shuffle rounds fold the four corner groups at the end.
//    Queries are visited in 2-D pixel patches per level when the queries are
//    the pixels themselves (encoder self-attention), so the overlapping
//    sampling neighbourhoods of a CTA hit in L1.
//
// Sampling-index arithmetic (bit-exact contract, SURVEY.md 8a-a17): the
// reference computes `loc * spatial - 0.5` with a double literal, so the
// product is rounded to fp32 BEFORE the subtraction; nvcc must not contract it
// into an FMA.  msda_geom() uses __fmul_rn/__fsub_rn and is shared by both
// kernels and by the index-dump entry point the parity tests use.
#include "msda_common.cuh"

// ---------------------------------------------------------------------------
// Strict kernel: reference mapping, reference order, no contraction.
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
msda_fwd_strict_kernel(const long long n, const T* __restrict__ value,
                       const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi,
                       const T* __restrict__ loc, const T* __restrict__ attw, T* __restrict__ out,
                       int S, int M, int D, int L, int Lq, int P) {
  __shared__ int s_h[MSDA_MAX_LEVELS], s_w[MSDA_MAX_LEVELS], s_start[MSDA_MAX_LEVELS];
  if (threadIdx.x < L) {
    s_h[threadIdx.x] = (int)shapes[2 * threadIdx.x];
    s_w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    s_start[threadIdx.x] = (int)lsi[threadIdx.x];
  }
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x; index < n; index += stride) {
    const int c = (int)(index % D);
    const long long pair = index / D;  // (b*Lq + q)*M + m
    const int m = (int)(pair % M);
    const long long b = pair / M / Lq;
    long long wptr = pair * L * P;
    const int qid_stride = M * D;
    const T* vb = value + b * (long long)S * qid_stride;
    T col = 0;
    for (int l = 0; l < L; ++l) {
      const int H = s_h[l], W = s_w[l];
      const T* vl = vb + (long long)s_start[l] * qid_stride + m * D + c;
      for (int p = 0; p < P; ++p, ++wptr) {
        const T lw_ = loc[2 * wptr], lh_ = loc[2 * wptr + 1];
        const T weight = attw[wptr];
        const MsdaGeom<T> g = msda_geom<T>(lw_, lh_, H, W);
        if (g.mask & 1) {
          const T hh = msda_sub((T)1, g.lh), hw = msda_sub((T)1, g.lw);
          const int w_stride = qid_stride, h_stride = W * qid_stride;
          const int o_hl = g.h_low * h_stride, o_wl = g.w_low * w_stride;
          T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
          if (g.mask & 2) v1 = vl[o_hl + o_wl];
          if (g.mask & 4) v2 = vl[o_hl + o_wl + w_stride];
          if (g.mask & 8) v3 = vl[o_hl + h_stride + o_wl];
          if (g.mask & 16) v4 = vl[o_hl + h_stride + o_wl + w_stride];
          const T w1 = msda_mul(hh, hw), w2 = msda_mul(hh, g.lw);
          const T w3 = msda_mul(g.lh, hw), w4 = msda_mul(g.lh, g.lw);
          T val = msda_mul(w1, v1);
          val = msda_add(val, msda_mul(w2, v2));
          val = msda_add(val, msda_mul(w3, v3));
          val = msda_add(val, msda_mul(w4, v4));
          col = msda_add(col, msda_mul(val, weight));
        }
      }
    }
    out[index] = col;
  }
}

// ---------------------------------------------------------------------------
// Index dump (parity instrumentation): (h_low, w_low, mask) per sample.
// ---------------------------------------------------------------------------
__global__ void msda_index_dump_kernel(long long n_samples, const int64_t* __restrict__ shapes,
                                       const float* __restrict__ loc, int32_t* __restrict__ out,
                                       int L, int P) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_samples; i += stride) {
    const int l = (int)((i / P) % L);
    const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
    const MsdaGeom<float> g = msda_geom<float>(loc[2 * i], loc[2 * i + 1], H, W);
    out[3 * i] = g.h_low; out[3 * i + 1] = g.w_low; out[3 * i + 2] = g.mask;
  }
}

// ---------------------------------------------------------------------------
// Fast warp kernel (fp32, D == 32, L*P <= 32).
// ---------------------------------------------------------------------------
// TH x TW query tile per CTA, NW warps; each warp owns TH*TW/NW queries.
// KC > 0: compile-time K = L*P (and PC = P) for the common GDINO shape; KC == 0: runtime.
// s_meta layout: [warp][corner][sample] of {byte offset, weight bits}, corner rows padded
// by 16 B so the four corner groups of a warp hit different banks on LDS.128.
constexpr int MSDA_META_ROW = 32 + 2;  // int2 per corner row (32 samples + pad)

// ValT = __nv_bfloat16 ("fast mode", SURVEY 8d cfg 2b): the module's value projection is a bf16 GEMM output; reading it
// in place halves the bytes every sample pulls through L1 (the kernel's real bound) and drops the fp32 upcast copy
// the reference makes (modeling_ov_grounding_dino_mask_dn.py:764).  A corner row is then 64 B = 4 x 16 B, so 16 lanes
// cover a sample and the two half-warps take the even / odd samples: half the gather instructions per (query, head).
// Arithmetic is unchanged (bf16 -> fp32 is exact, fp32 FMAs), so results equal the fp32 kernel on the upcast value.
template <int TH, int TW, int NW, int KC, int PC, typename OutT, typename ValT = float>
__global__ void __launch_bounds__(NW * 32)
msda_fwd_warp_kernel(const ValT* __restrict__ value, const int64_t* __restrict__ shapes,
                     const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                     const float* __restrict__ attw, OutT* __restrict__ out,
                     int S, int M, int L, int Lq, int P_rt, const __grid_constant__ MsdaTiling tl) {
  constexpr int D = 32;
  constexpr int TQ = TH * TW;
  constexpr int QPW = TQ / NW;  // queries per warp
  static_assert(TQ % NW == 0, "tile must split evenly over warps");
  __shared__ int s_h[MSDA_MAX_LEVELS], s_w[MSDA_MAX_LEVELS], s_start[MSDA_MAX_LEVELS];
  __shared__ __align__(16) int2 s_meta[NW][4][MSDA_META_ROW];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < L) {
    s_h[threadIdx.x] = (int)shapes[2 * threadIdx.x];
    s_w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    s_start[threadIdx.x] = (int)lsi[threadIdx.x];
  }
  __syncthreads();

  const int m = blockIdx.x % M;
  const int tile = blockIdx.x / M;
  const int b = blockIdx.y;
  const int P = KC > 0 ? PC : P_rt;
  const int K = KC > 0 ? KC : L * P_rt;
  const int G = (32 / K) < QPW ? (32 / K) : QPW;  // (query, head) pairs per phase-1 pass
  const int MD = M * D;

  // tile -> query mapping
  int lvl = 0, ty = 0, tx = 0;
  if (tl.mode == 1) {
    while (lvl + 1 < L && tile >= tl.tile_start[lvl + 1]) ++lvl;
    const int lt = tile - tl.tile_start[lvl];
    ty = lt / tl.tiles_w[lvl]; tx = lt % tl.tiles_w[lvl];
  }
  auto query_of = [&](int t) -> int {  // t: tile-local index; -1 if outside
    if (tl.mode == 0) { const int q = tile * TQ + t; return q < Lq ? q : -1; }
    const int py = ty * TH + t / TW, px = tx * TW + t % TW;
    if (py >= tl.H[lvl] || px >= tl.W[lvl]) return -1;
    return tl.q_start[lvl] + py * tl.W[lvl] + px;
  };

  constexpr bool HALF = sizeof(ValT) == 2;
  constexpr int VB = (int)sizeof(ValT);
  // fp32: lane = (corner[4], channel quad[8]); bf16: lane = (sample parity[2], corner[4], channel octet[4])
  const int corner = HALF ? ((lane >> 2) & 3) : (lane >> 3), cq = HALF ? (lane & 3) : (lane & 7);
  const int sp = lane >> 4;
  // per-lane base: batch, head and this lane's channel group folded in; meta offsets are bytes
  const char* vbl = reinterpret_cast<const char*>(value + (size_t)b * S * MD + m * D + cq * (HALF ? 8 : 4));
  const int g1 = lane / K, s1 = lane - g1 * K;  // phase-1 role of this lane
  const int l1 = s1 / P;

  for (int t0 = 0; t0 < QPW; t0 += G) {
    // ---- phase 1: one lane per sample ---------------------------------
    int q = -1;
    if (g1 < G && t0 + g1 < QPW) q = query_of(warp * QPW + t0 + g1);
    bool clean = true;   // all four corners of this lane's sample are in bounds
    {
      int2 meta[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) meta[c] = make_int2(-1, 0);
      if (q >= 0) {
        const size_t pair = ((size_t)b * Lq + q) * M + m;
        const size_t si = pair * K + s1;
        const float2 xy = ld_stream_f2(loc + 2 * si);
        const float aw = ld_stream_f1(attw + si);
        const int H = s_h[l1], W = s_w[l1];
        const MsdaGeom<float> ge = msda_geom<float>(xy.x, xy.y, H, W);
        clean = (ge.mask == 31);
        if (ge.mask & 1) {
          const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
          const int base = (s_start[l1] + ge.h_low * W + ge.w_low) * MD * VB;
          const float w1 = hh * hw, w2 = hh * ge.lw, w3 = ge.lh * hw, w4 = ge.lh * ge.lw;
          if (ge.mask & 2) meta[0] = make_int2(base, __float_as_int(w1 * aw));
          if (ge.mask & 4) meta[1] = make_int2(base + MD * VB, __float_as_int(w2 * aw));
          if (ge.mask & 8) meta[2] = make_int2(base + W * MD * VB, __float_as_int(w3 * aw));
          if (ge.mask & 16) meta[3] = make_int2(base + (W * MD + MD) * VB, __float_as_int(w4 * aw));
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) s_meta[warp][c][lane] = meta[c];
    }
    const unsigned dirty = __ballot_sync(0xffffffffu, !clean);
    __syncwarp();
    // ---- phase 2: lane = (corner, channel quad) -------------------------
    for (int g = 0; g < G && t0 + g < QPW; ++g) {
      const int qg = __shfl_sync(0xffffffffu, q, g * K);
      if (qg < 0) continue;  // warp-uniform
      const int2* mp = &s_meta[warp][corner][g * K];
      const unsigned gmask = (K >= 32 ? 0xffffffffu : ((1u << K) - 1u)) << (g * K);
      if constexpr (HALF) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        auto fma8 = [&](const uint4& raw, float w) {
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(h[i]);
            acc[2 * i] = fmaf(w, f.x, acc[2 * i]);
            acc[2 * i + 1] = fmaf(w, f.y, acc[2 * i + 1]);
          }
        };
        if (((dirty & gmask) == 0) && (K % 2 == 0)) {
          const int4* mp4 = reinterpret_cast<const int4*>(mp);
#pragma unroll (KC > 0 ? KC / 2 : 4)
          for (int s = 0; s < K / 2; ++s) {
            const int4 me = mp4[s];                       // samples 2s (x, y) and 2s + 1 (z, w) of this corner
            const int off = sp ? me.z : me.x;
            const float w = __int_as_float(sp ? me.w : me.y);
            fma8(__ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)off)), w);
          }
        } else {
          for (int s = sp; s < K; s += 2) {
            const int2 me = mp[s];
            if (me.x >= 0) fma8(__ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)me.x)), __int_as_float(me.y));
          }
        }
        // reduce-scatter over the 8 lanes holding the same 16-byte chunk (sample slot x corner): 4 + 2 + 1 shuffles
        // (same association order as msda_fwd_win_kernel, so both paths give bit-identical sums)
        float k4[4], k2[2];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float send = sp ? acc[j] : acc[j + 4];
          const float recv = __shfl_xor_sync(0xffffffffu, send, 16);
          k4[j] = (sp ? acc[j + 4] : acc[j]) + recv;
        }
        const int cb1 = corner >> 1, cb0 = corner & 1;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float send = cb1 ? k4[j] : k4[j + 2];
          const float recv = __shfl_xor_sync(0xffffffffu, send, 8);
          k2[j] = (cb1 ? k4[j + 2] : k4[j]) + recv;
        }
        const float send = cb0 ? k2[0] : k2[1];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 4);
        const float res = (cb0 ? k2[1] : k2[0]) + recv;
        OutT* op = out + (((size_t)b * Lq + qg) * M + m) * D + cq * 8 + sp * 4 + cb1 * 2 + cb0;
        if constexpr (sizeof(OutT) == 4) *op = res;
        else *op = __float2bfloat16(res);
        continue;
      }
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (((dirty & gmask) == 0) && (K % 2 == 0)) {
        // fast path: every corner of every sample of this pair is in bounds
        const int4* mp4 = reinterpret_cast<const int4*>(mp);
#pragma unroll (KC > 0 ? KC / 2 : 4)
        for (int s = 0; s < K / 2; ++s) {
          const int4 me = mp4[s];
          const float4 v0 = __ldg(reinterpret_cast<const float4*>(vbl + (unsigned)me.x));
          const float4 v1 = __ldg(reinterpret_cast<const float4*>(vbl + (unsigned)me.z));
          const float w0 = __int_as_float(me.y), w1 = __int_as_float(me.w);
          acc.x = fmaf(w0, v0.x, acc.x); acc.y = fmaf(w0, v0.y, acc.y);
          acc.z = fmaf(w0, v0.z, acc.z); acc.w = fmaf(w0, v0.w, acc.w);
          acc.x = fmaf(w1, v1.x, acc.x); acc.y = fmaf(w1, v1.y, acc.y);
          acc.z = fmaf(w1, v1.z, acc.z); acc.w = fmaf(w1, v1.w, acc.w);
        }
      } else {
#pragma unroll 2
        for (int s = 0; s < K; ++s) {
          const int2 me = mp[s];
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (me.x >= 0) v = __ldg(reinterpret_cast<const float4*>(vbl + (unsigned)me.x));
          const float w = __int_as_float(me.y);
          acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
          acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
        }
      }
      // reduce-scatter over the 4 corner groups: 2 + 1 shuffles, one channel per lane (same order as msda_win.cu)
      const int cb1 = corner >> 1, cb0 = corner & 1;
      float k2[2];
      {
        const float s0 = cb1 ? acc.x : acc.z, s1 = cb1 ? acc.y : acc.w;
        const float r0 = __shfl_xor_sync(0xffffffffu, s0, 16), r1 = __shfl_xor_sync(0xffffffffu, s1, 16);
        k2[0] = (cb1 ? acc.z : acc.x) + r0;
        k2[1] = (cb1 ? acc.w : acc.y) + r1;
      }
      const float send = cb0 ? k2[0] : k2[1];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 8);
      const float res = (cb0 ? k2[1] : k2[0]) + recv;
      OutT* op = out + (((size_t)b * Lq + qg) * M + m) * D + cq * 4 + cb1 * 2 + cb0;
      if constexpr (sizeof(OutT) == 4) *op = res;
      else *op = __float2bfloat16(res);
    }
    __syncwarp();
  }
}


// ---------------------------------------------------------------------------
// Paired-row fast mode (bf16 value).  The gather is bound by L1 wavefronts (one 128-byte line per warp-instruction
// slot), not by bytes: the four corners of a sample are four different lines in the reference layout, in fp32 (128 B
// rows) and in bf16 (64 B rows, half of every line wasted) alike.  msda_pack_pairs_kernel rewrites the bf16 value
// once per call into pairs[n][s][m][2][32]: slot 0 = value(s, m), slot 1 = value(s + 1, m) when pixel s + 1 lies in
// the same image row (else 0), i.e. both horizontal corners of a sample in ONE aligned 128-byte line.  A sample then
// costs two line fetches (rows h_low, h_low + 1) instead of four, and a warp instruction (32 x 16 B) covers two
// samples.  Lane = (sample parity, row, column, channel octet); per-corner weights are the same products as in
// msda_fwd_warp_kernel ((row weight * column weight) * attention weight), fp32 accumulation; corners outside the map
// read an all-zero line appended behind the last pixel with weight 0 (w_low == -1 re-bases the pair on pixel 0), so a
// NaN/Inf in a pixel the reference would not touch never reaches the sum.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
msda_pack_pairs_kernel(const __nv_bfloat16* __restrict__ value, __nv_bfloat16* __restrict__ pairs, long long n_chunks,
                       const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi, int S, int M, int L) {
  __shared__ int s_w[MSDA_MAX_LEVELS], s_start[MSDA_MAX_LEVELS];
  if (threadIdx.x < L) {
    s_w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    s_start[threadIdx.x] = (int)lsi[threadIdx.x];
  }
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x;
  if (blockIdx.x == 0 && threadIdx.x < 8)        // the all-zero line behind the last pixel: target of every off-map corner
    *reinterpret_cast<uint4*>(pairs + n_chunks * 8 + threadIdx.x * 8) = make_uint4(0u, 0u, 0u, 0u);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_chunks; i += stride) {
    const int oct = (int)(i & 3), slot = (int)((i >> 2) & 1);
    const long long pm = i >> 3;               // (n*S + s)*M + m
    const int m = (int)(pm % M);
    const long long ns = pm / M;
    const int sidx = (int)(ns % S);
    int l = 0;
    while (l + 1 < L && sidx >= s_start[l + 1]) ++l;
    const int w = (sidx - s_start[l]) % s_w[l];
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (slot == 0 || w + 1 < s_w[l])
      v = __ldg(reinterpret_cast<const uint4*>(value + ((ns + slot) * M + m) * 32 + oct * 8));
    *reinterpret_cast<uint4*>(pairs + i * 8) = v;
  }
}

constexpr int MSDA_PAIR_ROW = 32 + 2;   // int2 entries per (warp, row, column) slab: 32 samples + pad (slabs on different banks)

template <int TH, int TW, int NW, int KC, int PC, typename OutT>
__global__ void __launch_bounds__(NW * 32)
msda_fwd_pair_kernel(const __nv_bfloat16* __restrict__ pairs, const int64_t* __restrict__ shapes,
                     const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                     const float* __restrict__ attw, OutT* __restrict__ out,
                     int S, int M, int L, int Lq, int P_rt, const __grid_constant__ MsdaTiling tl) {
  constexpr int D = 32;
  constexpr int TQ = TH * TW;
  constexpr int QPW = TQ / NW;
  static_assert(TQ % NW == 0, "tile must split evenly over warps");
  __shared__ int s_h[MSDA_MAX_LEVELS], s_w[MSDA_MAX_LEVELS], s_start[MSDA_MAX_LEVELS];
  __shared__ __align__(16) int2 s_meta[NW][4][MSDA_PAIR_ROW];   // [row*2 + column]: {byte offset, weight bits}; off-map corner -> zero line

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < L) {
    s_h[threadIdx.x] = (int)shapes[2 * threadIdx.x];
    s_w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    s_start[threadIdx.x] = (int)lsi[threadIdx.x];
  }
  __syncthreads();

  const int m = blockIdx.x % M;
  const int tile = blockIdx.x / M;
  const int b = blockIdx.y;
  const int P = KC > 0 ? PC : P_rt;
  const int K = KC > 0 ? KC : L * P_rt;           // even (host-checked)
  const int G = (32 / K) < QPW ? (32 / K) : QPW;
  const int pix_bytes = M * 128;                  // one pixel of the pair tensor: M heads x (2 x 32 bf16)

  int lvl = 0, ty = 0, tx = 0;
  if (tl.mode == 1) {
    while (lvl + 1 < L && tile >= tl.tile_start[lvl + 1]) ++lvl;
    const int lt = tile - tl.tile_start[lvl];
    ty = lt / tl.tiles_w[lvl]; tx = lt % tl.tiles_w[lvl];
  }
  auto query_of = [&](int t) -> int {
    if (tl.mode == 0) { const int q = tile * TQ + t; return q < Lq ? q : -1; }
    const int py = ty * TH + t / TW, px = tx * TW + t % TW;
    if (py >= tl.H[lvl] || px >= tl.W[lvl]) return -1;
    return tl.q_start[lvl] + py * tl.W[lvl] + px;
  };

  // phase-2 role: lane = (sample parity, row, column, channel octet)
  const int sp = lane >> 4, r = (lane >> 3) & 1, col = (lane >> 2) & 1, oct = lane & 3;
  const char* vbl = reinterpret_cast<const char*>(pairs) + ((size_t)b * S * M + m) * 128 + (lane & 7) * 16;
  const int g1 = lane / K, s1 = lane - g1 * K;    // phase-1 role
  const int l1 = s1 / P;
  // byte offset (relative to this CTA's (batch, head) base) of the all-zero line behind the last pixel of the tensor
  const int zero_off = (int)(((long long)gridDim.y * S * M - ((long long)b * S * M + m)) * 128);

  for (int t0 = 0; t0 < QPW; t0 += G) {
    // ---- phase 1: one lane per sample -> two row entries ------------------
    int q = -1;
    if (g1 < G && t0 + g1 < QPW) q = query_of(warp * QPW + t0 + g1);
    {
      int2 e[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) e[c] = make_int2(zero_off, 0);   // weight 0 x zeros: contributes exactly 0
      if (q >= 0) {
        const size_t si = (((size_t)b * Lq + q) * M + m) * K + s1;
        const float2 xy = ld_stream_f2(loc + 2 * si);
        const float aw = ld_stream_f1(attw + si);
        const int H = s_h[l1], W = s_w[l1];
        const MsdaGeom<float> ge = msda_geom<float>(xy.x, xy.y, H, W);
        if (ge.mask & 1) {
          const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
          // column slots: pixel w_low (slot 0) and w_low + 1 (slot 1); w_low == -1 re-bases the pair on pixel 0,
          // whose slot 0 then carries the (h, w_high) corner
          const bool left_out = ge.w_low < 0;
          const int px = left_out ? 0 : ge.w_low;
          const bool col1 = !left_out && ge.w_low + 1 <= W - 1;
          const int off0 = (s_start[l1] + ge.h_low * W + px) * pix_bytes;
          const int off1 = off0 + W * pix_bytes;
          if (ge.h_low >= 0) {
            e[0] = make_int2(off0, __float_as_int((left_out ? hh * ge.lw : hh * hw) * aw));
            if (col1) e[1] = make_int2(off0, __float_as_int((hh * ge.lw) * aw));
          }
          if (ge.h_low + 1 <= H - 1) {
            e[2] = make_int2(off1, __float_as_int((left_out ? ge.lh * ge.lw : ge.lh * hw) * aw));
            if (col1) e[3] = make_int2(off1, __float_as_int((ge.lh * ge.lw) * aw));
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) s_meta[warp][c][lane] = e[c];
    }
    __syncwarp();
    // ---- phase 2: 2 samples x 2 rows x 128 B per warp instruction ----------
    for (int g = 0; g < G && t0 + g < QPW; ++g) {
      const int qg = __shfl_sync(0xffffffffu, q, g * K);
      if (qg < 0) continue;  // warp-uniform
      const int2* mp = &s_meta[warp][r * 2 + col][g * K + sp];
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      auto fma8 = [&](const uint4& raw, float w) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __bfloat1622float2(h[i]);
          acc[2 * i] = fmaf(w, f.x, acc[2 * i]);
          acc[2 * i + 1] = fmaf(w, f.y, acc[2 * i + 1]);
        }
      };
      if constexpr (KC > 0 && (KC / 2) % 4 == 0) {
        // batches of 4 line fetches in flight per lane, branch-free (predicated loads; an off corner contributes 0)
#pragma unroll
        for (int s0 = 0; s0 < KC / 2; s0 += 4) {
          int2 me[4]; uint4 raw[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) me[j] = mp[2 * (s0 + j)];
#pragma unroll
          for (int j = 0; j < 4; ++j) raw[j] = __ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)me[j].x));
#pragma unroll
          for (int j = 0; j < 4; ++j) fma8(raw[j], __int_as_float(me[j].y));
        }
      } else {
        for (int s = 0; s < K / 2; ++s) {
          const int2 me = mp[2 * s];
          fma8(__ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)me.x)), __int_as_float(me.y));
        }
      }
      // reduce-scatter over the 8 lanes that hold the same channel octet: 4 + 2 + 1 shuffles
      float k4[4], k2[2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float send = sp ? acc[j] : acc[j + 4];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 16);
        k4[j] = (sp ? acc[j + 4] : acc[j]) + recv;
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float send = r ? k4[j] : k4[j + 2];
        const float recv = __shfl_xor_sync(0xffffffffu, send, 8);
        k2[j] = (r ? k4[j + 2] : k4[j]) + recv;
      }
      const float send = col ? k2[0] : k2[1];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 4);
      const float res = (col ? k2[1] : k2[0]) + recv;
      const int ch = oct * 8 + sp * 4 + r * 2 + col;
      OutT* op = out + (((size_t)b * Lq + qg) * M + m) * D + ch;
      if constexpr (sizeof(OutT) == 4) *op = res;
      else *op = __float2bfloat16(res);
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// Backward (SURVEY 8f rank 1): grad_value (atomics), grad_sampling_loc, grad_attn_weight.
// Restates ms_deform_attn_col2im_bilinear + the col2im kernels (reference .cuh:66-124, 256-801): per output
// channel c of a (b, q, m) pair and per sample: top_grad_value = grad_out * weight; each in-bounds corner
// adds w_corner * top_grad_value to grad_value; grad_h/grad_w collect +-(other-axis weight) * v; the three
// per-sample scalars are then summed over the D channels.  One warp owns a pair: lanes stride over channels,
// three butterfly reductions per sample, lane 0 stores (each (b,q,m,l,p) has one owner, so no atomics there).
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_sum_t(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(256)
msda_bwd_warp_kernel(long long n_pairs, const T* __restrict__ value, const int64_t* __restrict__ shapes,
                     const int64_t* __restrict__ lsi, const T* __restrict__ loc, const T* __restrict__ attw,
                     const T* __restrict__ grad_out, T* __restrict__ grad_value, T* __restrict__ grad_loc,
                     T* __restrict__ grad_attw, int S, int M, int D, int L, int Lq, int P) {
  __shared__ int s_h[MSDA_MAX_LEVELS], s_w[MSDA_MAX_LEVELS], s_start[MSDA_MAX_LEVELS];
  if (threadIdx.x < L) {
    s_h[threadIdx.x] = (int)shapes[2 * threadIdx.x];
    s_w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    s_start[threadIdx.x] = (int)lsi[threadIdx.x];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long pair = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pair < n_pairs; pair += warps) {
    const int m = (int)(pair % M);
    const long long b = pair / M / Lq;
    const int qs = M * D;
    const long long vbase = b * (long long)S * qs + m * D;
    const T* go = grad_out + pair * D;
    long long wp = pair * L * P;
    for (int l = 0; l < L; ++l) {
      const int H = s_h[l], W = s_w[l];
      const long long lbase = vbase + (long long)s_start[l] * qs;
      for (int p = 0; p < P; ++p, ++wp) {
        const T weight = attw[wp];
        const MsdaGeom<T> g = msda_geom<T>(loc[2 * wp], loc[2 * wp + 1], H, W);
        T g_attn = 0, g_w = 0, g_h = 0;
        if (g.mask & 1) {
          const T hh = (T)1 - g.lh, hw = (T)1 - g.lw;
          const T w1 = hh * hw, w2 = hh * g.lw, w3 = g.lh * hw, w4 = g.lh * g.lw;
          const long long o1 = lbase + ((long long)g.h_low * W + g.w_low) * qs;
          const long long o2 = o1 + qs, o3 = o1 + (long long)W * qs, o4 = o3 + qs;
          for (int c = lane; c < D; c += 32) {
            const T tg = go[c];
            const T tgv = tg * weight;
            T v1 = 0, v2 = 0, v3 = 0, v4 = 0, gh = 0, gw = 0;
            if (g.mask & 2) { v1 = value[o1 + c]; gh -= hw * v1; gw -= hh * v1; atomicAdd(grad_value + o1 + c, w1 * tgv); }
            if (g.mask & 4) { v2 = value[o2 + c]; gh -= g.lw * v2; gw += hh * v2; atomicAdd(grad_value + o2 + c, w2 * tgv); }
            if (g.mask & 8) { v3 = value[o3 + c]; gh += hw * v3; gw -= g.lh * v3; atomicAdd(grad_value + o3 + c, w3 * tgv); }
            if (g.mask & 16) { v4 = value[o4 + c]; gh += g.lw * v4; gw += g.lh * v4; atomicAdd(grad_value + o4 + c, w4 * tgv); }
            g_attn += tg * (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
            g_w += (T)W * gw * tgv;
            g_h += (T)H * gh * tgv;
          }
        }
        g_attn = warp_sum_t(g_attn); g_w = warp_sum_t(g_w); g_h = warp_sum_t(g_h);
        if (lane == 0) {
          grad_attw[wp] = g_attn;
          grad_loc[2 * wp] = g_w;
          grad_loc[2 * wp + 1] = g_h;
        }
      }
    }
  }
}

template <typename T>
static int launch_bwd(const T* value, const int64_t* shapes, const int64_t* lsi, const T* loc, const T* attw,
                      const T* grad_out, T* grad_value, T* grad_loc, T* grad_attw, int N, int S, int M, int D, int L,
                      int Lq, int P, cudaStream_t st) {
  const long long pairs = (long long)N * Lq * M;
  if (pairs == 0) return VLLM_OK;
  long long blocks = (pairs + 7) / 8;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  msda_bwd_warp_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(pairs, value, shapes, lsi, loc, attw, grad_out, grad_value,
                                                             grad_loc, grad_attw, S, M, D, L, Lq, P);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

// ---------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------
// msda_win.cu: TMA-staged window kernel for the encoder shape; returns 1 when it does not apply.
template <typename ValT, typename OutT>
int msda_launch_window(const ValT* value, const int64_t* lsi, const float* loc, const float* attw, OutT* out, int N, int S,
                       int M, int L, int Lq, int P, const int64_t* host_shapes, cudaStream_t st);

static int g_msda_variant = 0;  // bench/tuning knob, see vllm_msda_set_variant

static bool build_tiling(MsdaTiling& tl, const int64_t* host_shapes, int L, int Lq, int S, int TH, int TW) {
  tl.mode = 0;
  tl.n_tiles = (Lq + TH * TW - 1) / (TH * TW);
  if (!host_shapes || Lq != S) return false;
  long long tot = 0; int tiles = 0;
  for (int l = 0; l < L; ++l) {
    const long long H = host_shapes[2 * l], W = host_shapes[2 * l + 1];
    if (H <= 0 || W <= 0 || H > INT_MAX || W > INT_MAX) return false;
    tl.H[l] = (int)H; tl.W[l] = (int)W; tl.q_start[l] = (int)tot;
    tl.tile_start[l] = tiles;
    tl.tiles_w[l] = (int)((W + TW - 1) / TW);
    tiles += tl.tiles_w[l] * (int)((H + TH - 1) / TH);
    tot += H * W;
  }
  tl.tile_start[L] = tiles;
  if (tot != Lq) return false;  // hint inconsistent with the query count: keep linear tiles
  tl.mode = 1; tl.n_tiles = tiles;
  return true;
}

template <int TH, int TW, int NW, typename OutT, typename ValT = float>
static int launch_warp(const ValT* value, const int64_t* shapes, const int64_t* lsi, const float* loc,
                       const float* attw, OutT* out, int N, int S, int M, int L, int Lq, int P,
                       const int64_t* host_shapes, cudaStream_t st) {
  MsdaTiling tl; memset(&tl, 0, sizeof(tl));
  build_tiling(tl, host_shapes, L, Lq, S, TH, TW);
  dim3 grid((unsigned)(tl.n_tiles * M), (unsigned)N);
  if (N > 65535) return VLLM_EUNSUPPORTED;
  if (L == 4 && P == 4)
    msda_fwd_warp_kernel<TH, TW, NW, 16, 4, OutT, ValT><<<grid, NW * 32, 0, st>>>(value, shapes, lsi, loc, attw, out,
                                                                                  S, M, L, Lq, P, tl);
  else
    msda_fwd_warp_kernel<TH, TW, NW, 0, 0, OutT, ValT><<<grid, NW * 32, 0, st>>>(value, shapes, lsi, loc, attw, out, S,
                                                                                 M, L, Lq, P, tl);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}


template <int TH, int TW, int NW, typename OutT>
static int launch_pair(const __nv_bfloat16* pairs, const int64_t* shapes, const int64_t* lsi, const float* loc,
                       const float* attw, OutT* out, int N, int S, int M, int L, int Lq, int P,
                       const int64_t* host_shapes, cudaStream_t st) {
  MsdaTiling tl; memset(&tl, 0, sizeof(tl));
  build_tiling(tl, host_shapes, L, Lq, S, TH, TW);
  dim3 grid((unsigned)(tl.n_tiles * M), (unsigned)N);
  if (N > 65535) return VLLM_EUNSUPPORTED;
  if (L == 4 && P == 4)
    msda_fwd_pair_kernel<TH, TW, NW, 16, 4, OutT><<<grid, NW * 32, 0, st>>>(pairs, shapes, lsi, loc, attw, out, S, M, L,
                                                                            Lq, P, tl);
  else
    msda_fwd_pair_kernel<TH, TW, NW, 0, 0, OutT><<<grid, NW * 32, 0, st>>>(pairs, shapes, lsi, loc, attw, out, S, M, L,
                                                                           Lq, P, tl);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

template <typename T>
static int launch_strict(const T* value, const int64_t* shapes, const int64_t* lsi, const T* loc, const T* attw,
                         T* out, int N, int S, int M, int D, int L, int Lq, int P, cudaStream_t st) {
  const long long n = (long long)N * Lq * M * D;
  if (n == 0) return VLLM_OK;
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  msda_fwd_strict_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(n, value, shapes, lsi, loc, attw, out, S, M, D, L,
                                                               Lq, P);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

static int check_common(const void* value, const void* shapes, const void* lsi, const void* loc, const void* attw,
                        const void* out, int N, int S, int M, int D, int L, int Lq, int P) {
  if (N < 0 || S < 0 || M <= 0 || D <= 0 || L <= 0 || Lq < 0 || P <= 0) return VLLM_EINVAL;
  if (L > MSDA_MAX_LEVELS) return VLLM_EUNSUPPORTED;
  if ((long long)N * Lq == 0) return VLLM_OK + 1000;  // empty: nothing to do
  if (!value || !shapes || !lsi || !loc || !attw || !out) return VLLM_EINVAL;
  if ((long long)S * M * D * 4 > INT_MAX) return VLLM_EUNSUPPORTED;  // per-image byte offsets are int32
  return VLLM_OK;
}

extern "C" {

int vllm_msda_set_variant(int v) { g_msda_variant = v; return VLLM_OK; }

int vllm_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                          const float* sampling_loc, const float* attn_weight, float* out, int batch,
                          int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                          int num_point, const int64_t* host_shapes_hint, int flags, void* stream) {
  int rc = check_common(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const bool strict = flags & 1;
  const int K = num_levels * num_point;
  if (!strict && channels == 32 && K <= 32 && vllm_aligned(value, 16) && vllm_aligned(out, 16) &&
      vllm_aligned(sampling_loc, 8)) {
    // encoder shape, fp32 rows: the TMA-staged window kernel (msda_win.cu) is opt-in (variant 33) -- 128-byte rows leave
    // room for an 8 x 8 patch only (not re-measured on the H100 against the global-memory patch kernel below);
    // bf16 rows (vllm_msda_forward_bf16v) take the window kernel by default
    if (g_msda_variant == 33) {
      const int r = msda_launch_window<float, float>(value, level_start_index, sampling_loc, attn_weight, out, batch,
                                                     spatial_size, num_heads, num_levels, num_query, num_point,
                                                     host_shapes_hint, st);
      if (r != 1) return r;
    }
    switch (g_msda_variant) {
      case 1: return launch_warp<8, 8, 8, float>(value, spatial_shapes, level_start_index, sampling_loc,
                                                 attn_weight, out, batch, spatial_size, num_heads, num_levels,
                                                 num_query, num_point, host_shapes_hint, st);
      case 2: return launch_warp<16, 16, 16, float>(value, spatial_shapes, level_start_index, sampling_loc,
                                                    attn_weight, out, batch, spatial_size, num_heads, num_levels,
                                                    num_query, num_point, host_shapes_hint, st);
      case 3: return launch_warp<16, 16, 32, float>(value, spatial_shapes, level_start_index, sampling_loc,
                                                    attn_weight, out, batch, spatial_size, num_heads, num_levels,
                                                    num_query, num_point, host_shapes_hint, st);
      case 4: return launch_warp<8, 8, 8, float>(value, spatial_shapes, level_start_index, sampling_loc,
                                                 attn_weight, out, batch, spatial_size, num_heads, num_levels,
                                                 num_query, num_point, nullptr, st);
      default:
        // few queries (decoder: 100 / 900 object queries): 128-query tiles leave most SMs idle and make every warp
        // walk 8 queries one HBM latency after the other -- 16-query tiles, 2 queries per warp, one pass
        if (num_query != spatial_size &&
            (long long)((num_query + 127) / 128) * num_heads * batch < 4ll * vllm_num_sms())
          return launch_warp<4, 4, 8, float>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out,
                                             batch, spatial_size, num_heads, num_levels, num_query, num_point, nullptr,
                                             st);
        return launch_warp<8, 16, 16, float>(value, spatial_shapes, level_start_index, sampling_loc,
                                             attn_weight, out, batch, spatial_size, num_heads, num_levels,
                                             num_query, num_point, host_shapes_hint, st);
    }
  }
  return launch_strict<float>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                              spatial_size, num_heads, channels, num_levels, num_query, num_point, st);
}

int vllm_msda_forward_bf16v(const void* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                            const float* sampling_loc, const float* attn_weight, void* out, int out_bf16, int batch,
                            int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                            int num_point, const int64_t* host_shapes_hint, void* stream) {
  int rc = check_common(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (channels != 32 || num_levels * num_point > 32) return VLLM_EUNSUPPORTED;   // caller upcasts and uses _f32
  if (!vllm_aligned(value, 16) || !vllm_aligned(out, 16) || !vllm_aligned(sampling_loc, 8)) return VLLM_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16* v = (const __nv_bfloat16*)value;
  if (g_msda_variant != 32) {                             // encoder shape: TMA-staged windows (msda_win.cu)
    const int r = out_bf16
        ? msda_launch_window<__nv_bfloat16, __nv_bfloat16>(v, level_start_index, sampling_loc, attn_weight,
                                                           (__nv_bfloat16*)out, batch, spatial_size, num_heads,
                                                           num_levels, num_query, num_point, host_shapes_hint, st)
        : msda_launch_window<__nv_bfloat16, float>(v, level_start_index, sampling_loc, attn_weight, (float*)out, batch,
                                                   spatial_size, num_heads, num_levels, num_query, num_point,
                                                   host_shapes_hint, st);
    if (r != 1) return r;
  }
  const bool few = num_query != spatial_size &&
                   (long long)((num_query + 127) / 128) * num_heads * batch < 4ll * vllm_num_sms();
  if (few && out_bf16)
    return launch_warp<4, 4, 8, __nv_bfloat16, __nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc,
                                                              attn_weight, (__nv_bfloat16*)out, batch, spatial_size,
                                                              num_heads, num_levels, num_query, num_point, nullptr, st);
  if (few)
    return launch_warp<4, 4, 8, float, __nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                                      (float*)out, batch, spatial_size, num_heads, num_levels,
                                                      num_query, num_point, nullptr, st);
  if (out_bf16)
    return launch_warp<8, 16, 16, __nv_bfloat16, __nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc,
                                                                attn_weight, (__nv_bfloat16*)out, batch, spatial_size,
                                                                num_heads, num_levels, num_query, num_point,
                                                                host_shapes_hint, st);
  return launch_warp<8, 16, 16, float, __nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                                      (float*)out, batch, spatial_size, num_heads, num_levels,
                                                      num_query, num_point, host_shapes_hint, st);
}

int vllm_msda_pack_pairs_bf16(const void* value, void* pairs, const int64_t* spatial_shapes,
                              const int64_t* level_start_index, int batch, int spatial_size, int num_heads,
                              int channels, int num_levels, void* stream) {
  if (batch < 0 || spatial_size < 0 || num_heads <= 0 || num_levels <= 0) return VLLM_EINVAL;
  if (channels != 32 || num_levels > MSDA_MAX_LEVELS) return VLLM_EUNSUPPORTED;
  const long long n_chunks = (long long)batch * spatial_size * num_heads * 8;
  if (n_chunks == 0) return VLLM_OK;
  if (!value || !pairs || !spatial_shapes || !level_start_index) return VLLM_EINVAL;
  if (!vllm_aligned(value, 16) || !vllm_aligned(pairs, 16)) return VLLM_EALIGN;
  long long blocks = (n_chunks + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  msda_pack_pairs_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)value, (__nv_bfloat16*)pairs, n_chunks, spatial_shapes, level_start_index, spatial_size,
      num_heads, num_levels);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_msda_forward_pairs(const void* pairs, const int64_t* spatial_shapes, const int64_t* level_start_index,
                            const float* sampling_loc, const float* attn_weight, void* out, int out_bf16, int batch,
                            int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                            int num_point, const int64_t* host_shapes_hint, void* stream) {
  int rc = check_common(pairs, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  const int K = num_levels * num_point;
  if (channels != 32 || K > 32 || (K & 1)) return VLLM_EUNSUPPORTED;
  if (((long long)batch * spatial_size * num_heads + 1) * 128 > INT_MAX) return VLLM_EUNSUPPORTED;  // zero line offset is int32
  if (!vllm_aligned(pairs, 128) || !vllm_aligned(sampling_loc, 8)) return VLLM_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16* v = (const __nv_bfloat16*)pairs;
  if (out_bf16)
    return launch_pair<8, 16, 16, __nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                                 (__nv_bfloat16*)out, batch, spatial_size, num_heads, num_levels,
                                                 num_query, num_point, host_shapes_hint, st);
  return launch_pair<8, 16, 16, float>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight, (float*)out,
                                       batch, spatial_size, num_heads, num_levels, num_query, num_point,
                                       host_shapes_hint, st);
}

int vllm_msda_forward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                          const double* sampling_loc, const double* attn_weight, double* out, int batch,
                          int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                          int num_point, void* stream) {
  int rc = check_common(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  return launch_strict<double>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, out, batch,
                               spatial_size, num_heads, channels, num_levels, num_query, num_point,
                               (cudaStream_t)stream);
}

int vllm_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                           const float* sampling_loc, const float* attn_weight, const float* grad_output,
                           float* grad_value, float* grad_sampling_loc, float* grad_attn_weight, int batch,
                           int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                           int num_point, void* stream) {
  int rc = check_common(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!grad_value || !grad_sampling_loc || !grad_attn_weight) return VLLM_EINVAL;
  return launch_bwd<float>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                           grad_value, grad_sampling_loc, grad_attn_weight, batch, spatial_size, num_heads, channels,
                           num_levels, num_query, num_point, (cudaStream_t)stream);
}

int vllm_msda_backward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                           const double* sampling_loc, const double* attn_weight, const double* grad_output,
                           double* grad_value, double* grad_sampling_loc, double* grad_attn_weight, int batch,
                           int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                           int num_point, void* stream) {
  int rc = check_common(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, batch,
                        spatial_size, num_heads, channels, num_levels, num_query, num_point);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!grad_value || !grad_sampling_loc || !grad_attn_weight) return VLLM_EINVAL;
  return launch_bwd<double>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                            grad_value, grad_sampling_loc, grad_attn_weight, batch, spatial_size, num_heads, channels,
                            num_levels, num_query, num_point, (cudaStream_t)stream);
}

int vllm_msda_sample_indices_f32(const int64_t* spatial_shapes, const float* sampling_loc, int32_t* out_hwm,
                                 long long n_samples, int num_levels, int num_point, void* stream) {
  if (n_samples < 0 || num_levels <= 0 || num_point <= 0) return VLLM_EINVAL;
  if (n_samples == 0) return VLLM_OK;
  if (!spatial_shapes || !sampling_loc || !out_hwm) return VLLM_EINVAL;
  long long blocks = (n_samples + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  msda_index_dump_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_samples, spatial_shapes,
                                                                             sampling_loc, out_hwm, num_levels,
                                                                             num_point);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // extern "C"
