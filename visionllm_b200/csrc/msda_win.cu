// TMA-staged multi-scale deformable attention forward for the ENCODER shape (queries == pixels, Lq == S).
//
// Replaces the same reference operator as msda.cu (mmcv ms_deform_attn_cuda_kernel.cuh:200-254 ==
// unipose/ops/src/cuda/ms_deform_im2col_cuda.cuh:237-300); entered from vllm_msda_forward_bf16v / _f32 when the
// caller's host-side shape hint proves that the queries are the pixels of the pyramid.
//
// Why: the gather is bound by L1 wavefronts, not by HBM bytes.  Through L1 a 64-byte bf16 row costs as much as a
// 128-byte fp32 row (one tag / one line per row); from shared memory it costs half.  (The rates behind this design were
// measured on another architecture and have not been re-measured on the H100.)
// So: one CTA owns a REGION of the image (a PH x PW patch of level-0 pixels and the pixels of every other level whose
// centres fall into the same normalised rectangle -- they all sample the same neighbourhoods) for ONE head, and
//   1. one thread TMA-loads (cp.async.bulk.tensor.5d, tensor = [D, M, W_l, H_l, N] per level, box = [D, 1, BW_l, BH_l, 1])
//      the bounded value window of every level into shared memory; coordinates outside the map are zero-filled by the
//      TMA unit, which IS the operator's zero padding (no per-corner predicates in the hot loop);
//   2. phase 1 (overlapping the TMA flight): one lane per (level, point) sample does the reference's index arithmetic
//      once (msda_geom, bit-exact) and writes {window byte offset, bilinear x attention weight} per corner;
//   3. phase 2: lane = (sample slot, corner, 16-byte chunk): LDS.128 from the window -- two horizontally adjacent
//      64-byte rows always cover complementary bank halves, so every quarter-warp is conflict-free -- fp32 FMAs,
//      a shuffle reduce-scatter (7 shuffles bf16 / 3 fp32) leaves one channel per lane, one coalesced 128-byte store;
//   4. a (query, head) with a sample outside its window (ballot) re-bases that pair on global memory and takes the
//      predicated path of msda.cu -- same arithmetic, so results do not depend on the window size.
// Arithmetic per corner is the one of msda_fwd_warp_kernel ((row weight x column weight) x attention weight, fp32
// FMAs): fast-mode tolerance class (<= 1e-5 max|ref| in fp32), indices bit-exact.
#include "msda_common.cuh"
#include "tc_common.cuh"
#include <string.h>

#define MSDA_WIN_LEVELS 4

struct MsdaWin {
  int L, PH, PW, RX, RY;
  int H[MSDA_WIN_LEVELS], W[MSDA_WIN_LEVELS];
  int q_start[MSDA_WIN_LEVELS];          // first query (== first pixel) of the level
  int BW[MSDA_WIN_LEVELS], BH[MSDA_WIN_LEVELS], halo[MSDA_WIN_LEVELS];
  int win_off[MSDA_WIN_LEVELS];          // byte offset of the level's window in dynamic shared memory
  int fill_tma;                          // bit l: level l's window arrives as a TMA box; else cooperative cp.async (see kernel)
  int px_cum[MSDA_WIN_LEVELS + 1];       // exclusive prefix sum of the window pixel counts BW * BH
  float inv_bw[MSDA_WIN_LEVELS];         // 1 / BW
  int zero_off;                          // a 128-byte all-zero row behind the windows: target of out-of-range samples
  int tx_bytes;                          // sum of the box bytes (what the mbarrier waits for)
};

struct MsdaWinMaps {
  CUtensorMap m[MSDA_WIN_LEVELS];
};

namespace {

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::
          "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// region boundary of level `l` along one axis: first pixel whose centre lies at or right of level-0 coordinate k*P,
// ceil((2kP*Wl - W0) / (2*W0)) clamped to [0, Wl]; 32-bit arithmetic (host checks W, H <= 16384 and k*P <= W0 + P)
__device__ __forceinline__ int region_bound(int k, int P, int Wl, int W0) {
  const unsigned num = 2u * (unsigned)(k * P) * (unsigned)Wl + (unsigned)W0 - 1u;   // n + d - 1 with n = 2kP*Wl - W0, d = 2*W0
  const unsigned b = num / (2u * (unsigned)W0);
  return b > (unsigned)Wl ? Wl : (int)b;
}

// 16-byte asynchronous copy global -> shared, zero-filled when `bytes` == 0 (the operator's zero padding)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}

constexpr int WIN_META_ROW = 32 + 2;    // int2 per corner row (32 samples + pad), as in msda_fwd_warp_kernel

}  // namespace

// Fused module input (QP = true; the GDINO deformable-attention MODULE rather than the bare operator, gd.py:706-784): the
// kernel takes the packed `sampling_offsets | attention_weights` projection output qp [N, Lq, ld] (bf16: M*K*2 offsets, then
// M*K logits) and the 2-d reference points [N, Lq, L, 2] (fp32) and does in phase 1 what the reference does in five
// elementwise torch kernels -- softmax over the K = 16 logits of a (query, head) (ATen's softmax_warp_forward: fp32 exp /
// butterfly sum / divide, result rounded to bf16), offset / (W_l, H_l) in bf16 (ATen div with the int64 normaliser cast to
// bf16), reference point + offset in fp32 -- bit for bit, then the same index arithmetic.  The attention weights the module
// returns are written as a side output.
struct MsdaQp {
  const __nv_bfloat16* qp;       // [N, Lq, ld]
  const float* ref;              // [N, Lq, L, 2]
  __nv_bfloat16* attw_out;       // [N, Lq, M, K] or null
  int ld, n_off;
};

// NW warps per CTA.  KC > 0: compile-time K = L*P (PC = P).
//
// The kernel is issue bound (~430 warp instructions per (query, head) against 64 data wavefronts), so the hot
// path is written for instruction count: everything that depends only on the lane's role (its sample's level: map and
// window geometry) lives in registers, the region's query list is a shared-memory table built once per CTA, global
// indices are 32-bit (host-checked), the bf16 rows are unpacked with one shift / one mask per element pair, and the
// per-corner metadata of a sample is one 8-byte shared load whose address carries the lane's sample parity.

template <typename ValT, typename OutT, int NW, int KC, int PC, bool QP = false>
__global__ void __launch_bounds__(NW * 32)
msda_fwd_win_kernel(const __grid_constant__ MsdaWinMaps maps, const ValT* __restrict__ value,
                    const int64_t* __restrict__ lsi, const float* __restrict__ loc, const float* __restrict__ attw,
                    OutT* __restrict__ out, int S, int M, int Lq, int P_rt, const __grid_constant__ MsdaWin wp,
                    const MsdaQp fq) {
  constexpr int D = 32;
  constexpr bool HALF = sizeof(ValT) == 2;
  constexpr int VB = (int)sizeof(ValT);
  constexpr int ROWB = D * VB;                             // bytes of one (pixel, head) row: 64 (bf16) / 128 (fp32)
  extern __shared__ __align__(128) unsigned char win[];
  __shared__ __align__(16) int2 s_meta[NW][4][WIN_META_ROW];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_bx0[MSDA_WIN_LEVELS], s_by0[MSDA_WIN_LEVELS], s_nx[MSDA_WIN_LEVELS], s_cum[MSDA_WIN_LEVELS + 1];
  __shared__ int s_ox[MSDA_WIN_LEVELS], s_oy[MSDA_WIN_LEVELS], s_start[MSDA_WIN_LEVELS];

  int* s_q = reinterpret_cast<int*>(win + wp.zero_off + 128);   // region-local index -> query (== pixel) index
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = wp.L;
  const int m = blockIdx.x % M;
  const int region = blockIdx.x / M;
  const int ky = region / wp.RX, kx = region - ky * wp.RX;
  const int b = blockIdx.y;
  const int P = KC > 0 ? PC : P_rt;
  const int K = KC > 0 ? KC : L * P_rt;
  const int G = 32 / K;                                    // (query, head) pairs per pass (K <= 32, host-checked)
  const int MD = M * D;

  if (warp == 0) {
    // lanes 0 .. L-1: the region's pixel ranges and window origin of one level each; lane 0 then issues the TMA loads
    int x0 = 0, y0 = 0, nx = 0, cnt = 0;
    if (lane < L) {
      x0 = region_bound(kx, wp.PW, wp.W[lane], wp.W[0]);
      y0 = region_bound(ky, wp.PH, wp.H[lane], wp.H[0]);
      nx = region_bound(kx + 1, wp.PW, wp.W[lane], wp.W[0]) - x0;
      cnt = nx * (region_bound(ky + 1, wp.PH, wp.H[lane], wp.H[0]) - y0);
      s_bx0[lane] = x0; s_by0[lane] = y0; s_nx[lane] = nx;
      s_ox[lane] = x0 - 1 - wp.halo[lane];
      s_oy[lane] = y0 - 1 - wp.halo[lane];
      s_start[lane] = (int)lsi[lane];
    }
    int cum = cnt;                                         // inclusive prefix sum over the (<= 4) level lanes
#pragma unroll
    for (int o = 1; o < MSDA_WIN_LEVELS; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, cum, o);
      if (lane >= o) cum += v;
    }
    if (lane < L) s_cum[lane + 1] = cum;
    if (lane == 0) {
      s_cum[0] = 0;
      if (wp.fill_tma) {
        const uint32_t bar0 = tc::smem_u32(&s_bar);
        tc::mbar_init(bar0, 1);
        tc::mbar_fence_init();
        tc::mbar_arrive_expect_tx(bar0, (uint32_t)wp.tx_bytes);
      }
    }
    __syncwarp();
    if (lane < L && ((wp.fill_tma >> lane) & 1))           // one TMA box per level (the init above is ordered by __syncwarp)
      tma_load_5d(tc::smem_u32(win + wp.win_off[lane]), &maps.m[lane], tc::smem_u32(&s_bar), 0, m, x0 - 1 - wp.halo[lane],
                  y0 - 1 - wp.halo[lane], b);
  }
  if (threadIdx.x >= 32 && threadIdx.x < 40)               // the zero row (never written by the TMA)
    *reinterpret_cast<uint4*>(win + wp.zero_off + (threadIdx.x - 32) * 16) = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  const int nq = s_cum[L];
  const uint32_t bar = tc::smem_u32(&s_bar);
  for (int t = threadIdx.x; t < nq; t += NW * 32) {        // the region's query list
    int lq = 0;
    while (lq + 1 < L && t >= s_cum[lq + 1]) ++lq;
    const int r = t - s_cum[lq];
    const int ry = r / s_nx[lq], rx = r - ry * s_nx[lq];
    s_q[t] = wp.q_start[lq] + (s_by0[lq] + ry) * wp.W[lq] + s_bx0[lq] + rx;
  }
  // Window fill.  fill_tma bit l set: level l arrives as one TMA box (issued above); the other levels are copied
  // cooperatively, one (pixel, head) row = ROWB / 16 cp.async of 16 bytes per thread and step, zero-filled outside the map
  // (the operator's zero padding).  A TMA box whose innermost run is one 64-byte row is request-rate bound, the
  // cooperative copy costs issue slots: the mix is a tuning knob (vllm_msda_set_window_fill), both fly while phase 1 of
  // the first pass runs.
  {
    constexpr int CPR = ROWB / 16;
    const uint32_t wbase = tc::smem_u32(win);
    const int total = wp.px_cum[L];
    for (int p = threadIdx.x; p < total; p += NW * 32) {
      int l = 0;
      while (l + 1 < L && p >= wp.px_cum[l + 1]) ++l;
      if ((wp.fill_tma >> l) & 1) continue;
      const int r = p - wp.px_cum[l];
      const int BWl = wp.BW[l];
      const int wy = (int)(((float)r + 0.5f) * wp.inv_bw[l]);       // r / BWl: exact for r < 2^16 (|error| << 0.5 / BWl)
      const int wx = r - wy * BWl;
      const int y = s_oy[l] + wy, x = s_ox[l] + wx;
      const bool ok = (unsigned)y < (unsigned)wp.H[l] && (unsigned)x < (unsigned)wp.W[l];
      const char* src = reinterpret_cast<const char*>(value + ((size_t)b * S + wp.q_start[l]) * MD + m * D);
      if (ok) src += ((size_t)y * wp.W[l] + x) * MD * VB;
      const uint32_t dst = wbase + wp.win_off[l] + r * ROWB;
#pragma unroll
      for (int cc = 0; cc < CPR; ++cc) cp_async16(dst + cc * 16, src + cc * 16, ok ? 16 : 0);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  __syncthreads();                                         // s_q complete
  bool landed = false;

  // phase-2 roles
  const int corner = HALF ? ((lane >> 2) & 3) : (lane >> 3), cq = HALF ? (lane & 3) : (lane & 7);
  const int sp = lane >> 4;
  const uint32_t wl = tc::smem_u32(win) + cq * 16;                             // this lane's 16-byte chunk of a window row
  const char* vbl = reinterpret_cast<const char*>(value + (size_t)b * S * MD + m * D) + cq * 16;   // global fallback
  const uint32_t meta_w = tc::smem_u32(&s_meta[warp][0][lane]);                // phase-1 store slot (corner rows 272 B apart)
  constexpr int META_ROWB = WIN_META_ROW * 8;
  // phase-1 roles: lane <-> sample s1 of pair g1; the sample's level l1 never changes, so its geometry sits in registers
  const int g1 = lane / K, s1 = lane - g1 * K;
  const int l1 = s1 / P;
  const int H1 = wp.H[l1], W1 = wp.W[l1];
  const int oy1 = s_oy[l1], ox1 = s_ox[l1];
  const int bh1 = wp.BH[l1] - 1, bw1 = wp.BW[l1] - 1;
  const int rowp1 = wp.BW[l1] * ROWB;
  const int woff1 = wp.win_off[l1];
  // batch / head / sample folded into the input bases: per-pass offsets are 32-bit (host-checked sizes)
  const float* loc_l = QP ? nullptr : loc + (((size_t)b * Lq * M + m) * K + s1) * 2;
  const float* attw_l = QP ? nullptr : attw + ((size_t)b * Lq * M + m) * K + s1;
  const __nv_bfloat16* qp_off = QP ? fq.qp + (size_t)b * Lq * fq.ld + (m * K + s1) * 2 : nullptr;
  const __nv_bfloat16* qp_lg = QP ? fq.qp + (size_t)b * Lq * fq.ld + fq.n_off + m * K + s1 : nullptr;
  const float* ref_l = QP ? fq.ref + ((size_t)b * Lq * L + l1) * 2 : nullptr;
  OutT* out_l = out + ((size_t)b * Lq * M + m) * D + (HALF ? cq * 8 + sp * 4 + (corner >> 1) * 2 + (corner & 1)
                                                          : cq * 4 + (corner >> 1) * 2 + (corner & 1));
  float Wb = 0.f, Hb = 0.f;
  if constexpr (QP) {
    Wb = __bfloat162float(__float2bfloat16_rn((float)W1));
    Hb = __bfloat162float(__float2bfloat16_rn((float)H1));
  }

  // per-lane inputs of one pass (this lane's sample of this lane's (query, head) pair), fetched one pass AHEAD so that the
  // global-memory latency of sampling_loc / attn_weight (or of the packed projection row) hides behind the gather
  struct Inp { int q; float a, b, c; uint32_t o2; };
  auto fetch = [&](int t0) -> Inp {
    Inp in; in.q = -1; in.a = in.b = in.c = 0.f; in.o2 = 0u;
    const int t = t0 + g1;
    if (g1 < G && t < nq) {
      in.q = s_q[t];
      if constexpr (QP) {
        const unsigned ro = (unsigned)in.q * (unsigned)fq.ld;
        in.o2 = *reinterpret_cast<const uint32_t*>(qp_off + ro);
        in.c = __bfloat162float(qp_lg[ro]);                                           // logit
        const float2 rp = *reinterpret_cast<const float2*>(ref_l + (unsigned)in.q * (unsigned)(L * 2));
        in.a = rp.x; in.b = rp.y;
      } else {
        const unsigned si = (unsigned)in.q * (unsigned)(M * K);
        const float2 xy = ld_stream_f2(loc_l + 2 * si);
        in.a = xy.x; in.b = xy.y;
        in.c = ld_stream_f1(attw_l + si);
      }
    }
    return in;
  };
  Inp nxt = fetch(warp * G);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();                                         // every thread's copies have landed and are visible to all
  if (wp.fill_tma) tc::mbar_wait(bar, 0);
  landed = true;

  for (int t0 = warp * G; t0 < nq; t0 += NW * G) {
    // ---- phase 1: one lane per sample ---------------------------------------------------------
    const Inp in = nxt;
    nxt = fetch(t0 + NW * G);                              // next pass's loads are in flight during this pass
    const int q = in.q;
    MsdaGeom<float> ge; ge.mask = 0; ge.h_low = 0; ge.w_low = 0; ge.lh = 0.f; ge.lw = 0.f;
    float aw = 0.f;
    bool in_win = true;
    {
      int2 meta[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) meta[c] = make_int2(wp.zero_off, 0);   // weight 0 x the zero row: contributes exactly 0,
                                                                         // and a NaN the reference never touches cannot leak
      float2 xy = make_float2(in.a, in.b);
      if constexpr (QP) {
        // every lane takes part in the softmax shuffles (idle lanes carry logit 0); K == 16: two pairs per warp
        const float lg = in.c;
        float mx = lg;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float e = expf(lg - mx);
        float sum = e;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const __nv_bfloat16 wb = __float2bfloat16_rn(e / sum);
        aw = __bfloat162float(wb);
        if (q >= 0) {
          if (fq.attw_out) fq.attw_out[(((size_t)b * Lq + q) * M + m) * K + s1] = wb;
          const __nv_bfloat162 ob = *reinterpret_cast<const __nv_bfloat162*>(&in.o2);
          const float ox = __bfloat162float(__float2bfloat16_rn(__fdiv_rn(__low2float(ob), Wb)));
          const float oy = __bfloat162float(__float2bfloat16_rn(__fdiv_rn(__high2float(ob), Hb)));
          xy = make_float2(__fadd_rn(in.a, ox), __fadd_rn(in.b, oy));
        }
      } else {
        aw = in.c;
      }
      if (q >= 0) {
        ge = msda_geom<float>(xy.x, xy.y, H1, W1);
        if (ge.mask & 1) {
          const int wy = ge.h_low - oy1, wx = ge.w_low - ox1;
          in_win = ((unsigned)wy < (unsigned)bh1) && ((unsigned)wx < (unsigned)bw1);
          const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
          const int base = woff1 + wy * rowp1 + wx * ROWB;
          // corners outside the MAP but inside the window read TMA zero fill: no predicate needed
          meta[0] = make_int2(base, __float_as_int((hh * hw) * aw));
          meta[1] = make_int2(base + ROWB, __float_as_int((hh * ge.lw) * aw));
          meta[2] = make_int2(base + rowp1, __float_as_int((ge.lh * hw) * aw));
          meta[3] = make_int2(base + rowp1 + ROWB, __float_as_int((ge.lh * ge.lw) * aw));
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c)
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(meta_w + c * META_ROWB), "r"(meta[c].x), "r"(meta[c].y) : "memory");
    }
    const unsigned outside = __ballot_sync(0xffffffffu, !in_win);
    __syncwarp();
    // ---- phase 2 --------------------------------------------------------------------------------
    for (int g = 0; g < G; ++g) {
      const int qg = __shfl_sync(0xffffffffu, q, g * K);
      if (qg < 0) continue;                                // warp-uniform
      const unsigned gmask = (K >= 32 ? 0xffffffffu : ((1u << K) - 1u)) << (g * K);
      const bool dirty = (outside & gmask) != 0;           // warp-uniform
      if (dirty) {
        // re-base this pair on global memory: byte offsets relative to vbl, -1 for a corner outside the map
        __syncwarp();
        if (g1 == g) {
          int2 meta[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) meta[c] = make_int2(-1, 0);
          if (ge.mask & 1) {
            const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
            const int base = (s_start[l1] + ge.h_low * W1 + ge.w_low) * MD * VB;
            if (ge.mask & 2) meta[0] = make_int2(base, __float_as_int((hh * hw) * aw));
            if (ge.mask & 4) meta[1] = make_int2(base + MD * VB, __float_as_int((hh * ge.lw) * aw));
            if (ge.mask & 8) meta[2] = make_int2(base + W1 * MD * VB, __float_as_int((ge.lh * hw) * aw));
            if (ge.mask & 16) meta[3] = make_int2(base + (W1 * MD + MD) * VB, __float_as_int((ge.lh * ge.lw) * aw));
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) s_meta[warp][c][lane] = meta[c];
        }
        __syncwarp();
      }
      const int2* mp = &s_meta[warp][corner][g * K];
      const int2* mph = mp + sp;                           // bf16 rows: the lane's sample parity rides in the address
      const int4* mp4 = reinterpret_cast<const int4*>(mp);
      OutT* op = out_l + (size_t)((unsigned)qg * (unsigned)MD);
      if constexpr (HALF) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        auto fma8 = [&](const uint4& raw, float w) {       // bf16 -> fp32 is a shift (low half) / a mask (high half)
          const uint32_t words[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            acc[2 * i] = fmaf(w, __uint_as_float(words[i] << 16), acc[2 * i]);
            acc[2 * i + 1] = fmaf(w, __uint_as_float(words[i] & 0xffff0000u), acc[2 * i + 1]);
          }
        };
        if (!dirty && (K % 2 == 0)) {
#pragma unroll (KC > 0 ? KC / 2 : 4)
          for (int s = 0; s < K / 2; ++s) {
            const int2 me = mph[2 * s];                    // sample 2s + sp of this corner: one 8-byte broadcast load
            fma8(lds128(wl + me.x), __int_as_float(me.y));
          }
        } else if (!dirty) {
          for (int s = sp; s < K; s += 2) {
            const int2 me = mp[s];
            fma8(lds128(wl + me.x), __int_as_float(me.y));
          }
        } else {
          for (int s = sp; s < K; s += 2) {
            const int2 me = mp[s];
            if (me.x >= 0) fma8(__ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)me.x)), __int_as_float(me.y));
          }
        }
        // reduce-scatter over the 8 lanes holding the same 16-byte chunk (sample slot x corner): 4 + 2 + 1 shuffles
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
        if constexpr (sizeof(OutT) == 4) *op = res;
        else *op = __float2bfloat16(res);
      } else {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        auto fma4 = [&](const uint4& v, float w) {
          acc.x = fmaf(w, __uint_as_float(v.x), acc.x); acc.y = fmaf(w, __uint_as_float(v.y), acc.y);
          acc.z = fmaf(w, __uint_as_float(v.z), acc.z); acc.w = fmaf(w, __uint_as_float(v.w), acc.w);
        };
        if (!dirty && (K % 2 == 0)) {
#pragma unroll (KC > 0 ? KC / 2 : 4)
          for (int s = 0; s < K / 2; ++s) {
            const int4 me = mp4[s];                        // samples 2s (x, y) and 2s + 1 (z, w) of this corner
            const uint4 v0 = lds128(wl + me.x), v1 = lds128(wl + me.z);
            fma4(v0, __int_as_float(me.y));
            fma4(v1, __int_as_float(me.w));
          }
        } else if (!dirty) {
          for (int s = 0; s < K; ++s) {
            const int2 me = mp[s];
            fma4(lds128(wl + me.x), __int_as_float(me.y));
          }
        } else {
          for (int s = 0; s < K; ++s) {
            const int2 me = mp[s];
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (me.x >= 0) v = __ldg(reinterpret_cast<const uint4*>(vbl + (unsigned)me.x));
            fma4(v, __int_as_float(me.y));
          }
        }
        // reduce-scatter over the 4 corner groups: 2 + 1 shuffles, one channel per lane
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
        if constexpr (sizeof(OutT) == 4) *op = res;
        else *op = __float2bfloat16(res);
      }
    }
    __syncwarp();
  }
  if (!landed && wp.fill_tma) tc::mbar_wait(bar, 0);       // never leave with a TMA in flight into this CTA's smem
}

// ---------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------
static int g_win_ph = 0, g_win_pw = 0, g_win_halo = 0;      // 0: defaults; bench / tuning knob (vllm_msda_set_window)
static int g_win_fill_tma = -1;   // vllm_msda_set_window_fill: bit l = level l by TMA box; 0 = all cp.async; 1 = (legacy) all TMA; < 0 default

extern "C" int vllm_msda_set_window(int patch_h, int patch_w, int halo0) {
  if (patch_h < 0 || patch_w < 0 || halo0 < 0) return VLLM_EINVAL;
  g_win_ph = patch_h; g_win_pw = patch_w; g_win_halo = halo0;
  return VLLM_OK;
}

extern "C" int vllm_msda_set_window_fill(int tma) {
  g_win_fill_tma = tma == 1 ? (1 << MSDA_WIN_LEVELS) - 1 : tma;     // 1 keeps its r2 meaning: every level by TMA
  return VLLM_OK;
}

constexpr int WIN_FILL_DEFAULT_BF16 = (1 << MSDA_WIN_LEVELS) - 1;   // every level staged; not re-tuned for the H100
constexpr int WIN_FILL_DEFAULT_F32 = (1 << MSDA_WIN_LEVELS) - 1;

static void set_fill(MsdaWin& wp, int vb) {
  int mask = g_win_fill_tma >= 0 ? g_win_fill_tma : (vb == 2 ? WIN_FILL_DEFAULT_BF16 : WIN_FILL_DEFAULT_F32);
  mask &= (1 << wp.L) - 1;
  wp.fill_tma = mask;
  wp.tx_bytes = 0;
  for (int l = 0; l < wp.L; ++l)
    if ((mask >> l) & 1) wp.tx_bytes += wp.BW[l] * wp.BH[l] * 32 * vb;
}

struct WinCacheEntry {
  const void* value; int N, S, M, L, vb; int64_t shapes[2 * MSDA_WIN_LEVELS]; int ph, pw, halo;
  MsdaWinMaps maps; MsdaWin wp; int smem; bool ok;
};
static WinCacheEntry g_win_cache[8];
static int g_win_cache_next = 0;

template <typename ValT>
static bool build_window(WinCacheEntry& e, const ValT* value, const int64_t* hs, int N, int S, int M, int L) {
  constexpr int VB = (int)sizeof(ValT);
  constexpr int ROWB = 32 * VB;
  MsdaWin& wp = e.wp;
  memset(&wp, 0, sizeof(wp));
  wp.L = L;
  long long tot = 0;
  for (int l = 0; l < L; ++l) {
    const long long H = hs[2 * l], W = hs[2 * l + 1];
    if (H <= 0 || W <= 0 || H > 16384 || W > 16384) return false;
    wp.H[l] = (int)H; wp.W[l] = (int)W; wp.q_start[l] = (int)tot;
    tot += H * W;
  }
  if (tot != S) return false;
  // level-0 patch: 16 x 32 pixels for bf16 rows (64 B): 159 KB of windows, one 32-warp CTA per SM (the halo is
  // amortised over 4x the queries of an 8 x 16 patch; the choice has not been re-swept on the H100); 8 x 8 for fp32 rows
  // (128 B): 95 KB, two 16-warp CTAs per SM
  wp.PH = g_win_ph > 0 ? g_win_ph : (VB == 2 ? 16 : 8);
  wp.PW = g_win_pw > 0 ? g_win_pw : (VB == 2 ? 32 : 8);
  const int halo0 = g_win_halo > 0 ? g_win_halo : (VB == 2 ? 8 : 6);
  wp.RX = (wp.W[0] + wp.PW - 1) / wp.PW;
  wp.RY = (wp.H[0] + wp.PH - 1) / wp.PH;
  int off = 0;
  for (int l = 0; l < L; ++l) {
    // offsets are predicted in pixels of the sampled level: keep a few pixels of halo on the coarse levels too
    const int min_halo = VB == 2 ? 3 : 2;
    int halo = (int)((halo0 * (long long)wp.W[l] + wp.W[0] - 1) / wp.W[0]);
    if (halo < min_halo) halo = min_halo;
    if (l == 0) halo = halo0;
    wp.halo[l] = halo;
    wp.BW[l] = (int)((wp.PW * (long long)wp.W[l] + wp.W[0] - 1) / wp.W[0]) + 2 + 2 * halo;
    wp.BH[l] = (int)((wp.PH * (long long)wp.H[l] + wp.H[0] - 1) / wp.H[0]) + 2 + 2 * halo;
    if (wp.BW[l] > 256 || wp.BH[l] > 256 || wp.BW[l] * wp.BH[l] > 65535) return false;
    wp.win_off[l] = off;
    const int bytes = wp.BW[l] * wp.BH[l] * ROWB;
    wp.px_cum[l + 1] = wp.px_cum[l] + wp.BW[l] * wp.BH[l];
    wp.inv_bw[l] = 1.0f / (float)wp.BW[l];
    off += (bytes + 127) & ~127;
  }
  wp.zero_off = off;
  off += 128;
  long long nq_max = 0;                                      // upper bound of a region's query count (the s_q table behind the zero row)
  for (int l = 0; l < L; ++l)
    nq_max += ((wp.PW * (long long)wp.W[l] + wp.W[0] - 1) / wp.W[0] + 1) * ((wp.PH * (long long)wp.H[l] + wp.H[0] - 1) / wp.H[0] + 1);
  off += (int)((nq_max * 4 + 127) & ~127ll);
  if (nq_max > 8192 || off > 190 * 1024) return false;     // > 110 KB: one CTA of 32 warps per SM instead of two of 16
  e.smem = off;
  PFN_cuTensorMapEncodeTiled_v12000 enc = vllm_tma_encoder();
  if (!enc) return false;
  for (int l = 0; l < L; ++l) {
    const size_t MD = (size_t)M * 32;
    cuuint64_t dims[5] = {32, (cuuint64_t)M, (cuuint64_t)wp.W[l], (cuuint64_t)wp.H[l], (cuuint64_t)N};
    cuuint64_t strides[4] = {(cuuint64_t)32 * VB, MD * VB, (cuuint64_t)wp.W[l] * MD * VB, (cuuint64_t)S * MD * VB};
    cuuint32_t box[5] = {32, 1, (cuuint32_t)wp.BW[l], (cuuint32_t)wp.BH[l], 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    const ValT* base = value + (size_t)wp.q_start[l] * MD;
    CUresult r = enc(&e.maps.m[l], VB == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5,
                     const_cast<ValT*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return false;
  }
  return true;
}

template <typename ValT>
static const WinCacheEntry* window_for(const ValT* value, const int64_t* hs, int N, int S, int M, int L) {
  for (auto& e : g_win_cache)
    if (e.ok && e.value == value && e.N == N && e.S == S && e.M == M && e.L == L && e.vb == (int)sizeof(ValT) &&
        e.ph == g_win_ph && e.pw == g_win_pw && e.halo == g_win_halo && memcmp(e.shapes, hs, 2 * L * sizeof(int64_t)) == 0)
      return &e;
  WinCacheEntry& e = g_win_cache[g_win_cache_next];
  g_win_cache_next = (g_win_cache_next + 1) % 8;
  e.ok = false;
  e.value = value; e.N = N; e.S = S; e.M = M; e.L = L; e.vb = (int)sizeof(ValT);
  e.ph = g_win_ph; e.pw = g_win_pw; e.halo = g_win_halo;
  memcpy(e.shapes, hs, 2 * L * sizeof(int64_t));
  if (!build_window<ValT>(e, value, hs, N, S, M, L)) return nullptr;
  e.ok = true;
  return &e;
}

// Returns VLLM_OK after a launch, 1 when the window path does not apply (caller falls back), or an error.
template <typename ValT, typename OutT>
int msda_launch_window(const ValT* value, const int64_t* lsi, const float* loc, const float* attw, OutT* out, int N, int S,
                       int M, int L, int Lq, int P, const int64_t* host_shapes, cudaStream_t st) {
  constexpr int NW = 16;
  if (!host_shapes || Lq != S || L > MSDA_WIN_LEVELS || L * P > 32 || N > 65535) return 1;
  const WinCacheEntry* e = window_for<ValT>(value, host_shapes, N, S, M, L);
  if (!e) return 1;
  dim3 grid((unsigned)(e->wp.RX * e->wp.RY * M), (unsigned)N);
  const bool big = e->smem > 110 * 1024;                   // one 32-warp CTA per SM (tuning knob territory)
  auto launch = [&](auto kern, int nw) -> int {
    static int configured = -1;
    if (configured < e->smem) {
      const int want = big ? e->smem : 112 * 1024;
      cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, want);
      if (err != cudaSuccess) return (int)err;
      configured = want;
    }
    MsdaWin wp = e->wp;
    set_fill(wp, (int)sizeof(ValT));
    kern<<<grid, nw * 32, e->smem, st>>>(e->maps, value, lsi, loc, attw, out, S, M, Lq, P, wp, MsdaQp{});
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  };
  if (L == 4 && P == 4) return big ? launch(msda_fwd_win_kernel<ValT, OutT, 32, 16, 4>, 32) : launch(msda_fwd_win_kernel<ValT, OutT, NW, 16, 4>, NW);
  if (big) return 1;
  return launch(msda_fwd_win_kernel<ValT, OutT, NW, 0, 0>, NW);
}

// fused module input (bf16 value, K == 16 only); returns 1 when the window path does not apply
template <typename OutT>
static int launch_window_qp(const __nv_bfloat16* value, const int64_t* lsi, const MsdaQp& fq, OutT* out, int N, int S, int M, int L,
                            int Lq, int P, const int64_t* host_shapes, cudaStream_t st) {
  if (!host_shapes || Lq != S || L != 4 || P != 4 || N > 65535) return 1;
  const WinCacheEntry* e = window_for<__nv_bfloat16>(value, host_shapes, N, S, M, L);
  if (!e) return 1;
  dim3 grid((unsigned)(e->wp.RX * e->wp.RY * M), (unsigned)N);
  const bool big = e->smem > 110 * 1024;
  auto launch = [&](auto kern, int nw) -> int {
    static int configured = -1;
    if (configured < e->smem) {
      const int want = big ? e->smem : 112 * 1024;
      cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, want);
      if (err != cudaSuccess) return (int)err;
      configured = want;
    }
    MsdaWin wp = e->wp;
    set_fill(wp, 2);
    kern<<<grid, nw * 32, e->smem, st>>>(e->maps, value, lsi, nullptr, nullptr, out, S, M, Lq, P, wp, fq);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  };
  return big ? launch(msda_fwd_win_kernel<__nv_bfloat16, OutT, 32, 16, 4, true>, 32)
             : launch(msda_fwd_win_kernel<__nv_bfloat16, OutT, 16, 16, 4, true>, 16);
}

extern "C" int vllm_msda_forward_fused_bf16(const void* value, const int64_t* level_start_index, const void* qp, int ld_qp,
                                            const float* reference_points, void* out, int out_bf16, void* attn_weights_out,
                                            int batch, int spatial_size, int num_heads, int channels, int num_levels,
                                            int num_query, int num_point, const int64_t* host_shapes_hint, void* stream) {
  if (batch < 0 || spatial_size <= 0 || num_heads <= 0 || num_query < 0) return VLLM_EINVAL;
  if ((long long)batch * num_query == 0) return VLLM_OK;
  if (!value || !level_start_index || !qp || !reference_points || !out) return VLLM_EINVAL;
  const int K = num_levels * num_point;
  if (channels != 32 || num_levels != 4 || num_point != 4 || ld_qp < num_heads * K * 3 || (ld_qp & 1)) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(value, 16) || !vllm_aligned(qp, 4) || !vllm_aligned(reference_points, 8)) return VLLM_EALIGN;
  if ((long long)spatial_size * num_heads * channels * 4 > INT_MAX) return VLLM_EUNSUPPORTED;
  if ((long long)num_query * ld_qp > UINT_MAX) return VLLM_EUNSUPPORTED;     // 32-bit row offsets inside one image
  MsdaQp fq{(const __nv_bfloat16*)qp, reference_points, (__nv_bfloat16*)attn_weights_out, ld_qp, num_heads * K * 2};
  cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16* v = (const __nv_bfloat16*)value;
  const int r = out_bf16 ? launch_window_qp<__nv_bfloat16>(v, level_start_index, fq, (__nv_bfloat16*)out, batch, spatial_size,
                                                           num_heads, num_levels, num_query, num_point, host_shapes_hint, st)
                         : launch_window_qp<float>(v, level_start_index, fq, (float*)out, batch, spatial_size, num_heads,
                                                   num_levels, num_query, num_point, host_shapes_hint, st);
  return r == 1 ? VLLM_EUNSUPPORTED : r;
}

template int msda_launch_window<float, float>(const float*, const int64_t*, const float*, const float*, float*, int, int, int,
                                              int, int, int, const int64_t*, cudaStream_t);
template int msda_launch_window<__nv_bfloat16, float>(const __nv_bfloat16*, const int64_t*, const float*, const float*, float*,
                                                      int, int, int, int, int, int, const int64_t*, cudaStream_t);
template int msda_launch_window<__nv_bfloat16, __nv_bfloat16>(const __nv_bfloat16*, const int64_t*, const float*, const float*,
                                                              __nv_bfloat16*, int, int, int, int, int, int, const int64_t*,
                                                              cudaStream_t);
