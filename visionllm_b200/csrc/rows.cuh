// Register-resident bf16 rows: the 16-byte vector format, the row reduction and the RMSNorm / LayerNorm steps shared by
// the row kernels (fused_ops.cu, seqglue.cu, train_ops.cu, peer.cu, dwconv.cu, groupnorm.cu).
//
// A row of `cols` bf16 is nvec = cols / 8 16-byte vectors.  It is owned by TPR consecutive threads (a warp, several
// warps or the whole CTA); thread tr = threadIdx.x % TPR holds vectors tr, tr + TPR, ..., VPT of them, zero past nvec.
// The reduction order is part of each kernel's output bits: a per-thread chain over its vectors in order, the warp's
// xor-shuffle tree, then the warps of the row in warp order.
#pragma once
#include "common.cuh"
#include <math.h>
#include <type_traits>

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// Sum (MAX: maximum) of v over the TPR threads of a row; every one of them gets the result.  For TPR > 32 the warp
// partials go through sh (one float per warp of the CTA) between barriers; the first barrier waits until the previous
// reduction through sh has been read, so a caller that alternates between two sh buffers passes WAIT = false.  NT, the
// threads of the CTA, defaults to one row per CTA; then the row's partials sit at constant offsets of sh.
template <int TPR, bool MAX = false, bool WAIT = true, int NT = TPR>
__device__ __forceinline__ float row_reduce(float v, float* sh) {
  v = MAX ? warp_max(v) : warp_sum(v);
  if constexpr (TPR > 32) {
    constexpr int WPR = TPR / 32;                      // warps per row
    const int w = threadIdx.x >> 5, first = NT == TPR ? 0 : w / WPR * WPR;
    if (WAIT) __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[w] = v;
    __syncthreads();
    float t = MAX ? -INFINITY : 0.f;
#pragma unroll
    for (int i = 0; i < WPR; ++i) t = MAX ? fmaxf(t, sh[first + i]) : t + sh[first + i];
    v = t;
  }
  return v;
}
template <int TPR, bool WAIT = true, int NT = TPR>
__device__ __forceinline__ float row_sum(float v, float* sh) { return row_reduce<TPR, false, WAIT, NT>(v, sh); }
template <int TPR>
__device__ __forceinline__ float row_max(float v, float* sh) { return row_reduce<TPR, true>(v, sh); }

// RMSNorm (HF LlamaRMSNorm): rstd = rsqrt(mean(x^2) + eps) of the row, then y = w * bf16(x * rstd) -- the input-dtype
// rounding before the weight is the reference's, so both bf16 roundings are kept.
template <int VPT, int TPR, bool WAIT = true, int NT = TPR>
__device__ __forceinline__ float rms_rstd(const uint4 (&x)[VPT], int cols, float eps, float* sh) {
  const int tr = threadIdx.x % TPR, nvec = cols / 8;
  float s2 = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    if (tr + i * TPR < nvec) {
      float f[8]; unpack8(x[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s2 += f[j] * f[j];
    }
  }
  return rsqrtf(row_sum<TPR, WAIT, NT>(s2, sh) / cols + eps);
}
// x is vector v of the row; the weight vector is read from w here, after x is unpacked (ptxas allocates fewer registers
// for that order than for a weight loaded ahead of the call).
__device__ __forceinline__ uint4 rms_apply(const uint4& x, const __nv_bfloat16* __restrict__ w, int v, float rstd) {
  float f[8], wv[8], o[8];
  unpack8(x, f); unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = wv[j] * __bfloat162float(__float2bfloat16(f[j] * rstd));
  return pack8(o);
}

// LayerNorm (nn.LayerNorm): fp32 mean, then the variance in a second pass over the register-resident row;
// returns (mean, rstd).  y = (x - mean) * rstd * w + b in fp32, for vector v of the row as rms_apply.
template <int VPT, int TPR, int NT = TPR>
__device__ __forceinline__ float2 ln_stats(const uint4 (&x)[VPT], int cols, float eps, float* sh) {
  const int tr = threadIdx.x % TPR, nvec = cols / 8;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    if (tr + i * TPR < nvec) {
      float f[8]; unpack8(x[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[j];
    }
  }
  const float mean = row_sum<TPR, true, NT>(s, sh) / cols;
  float d2 = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    if (tr + i * TPR < nvec) {
      float f[8]; unpack8(x[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; d2 += d * d; }
    }
  }
  return make_float2(mean, rsqrtf(row_sum<TPR, true, NT>(d2, sh) / cols + eps));
}
__device__ __forceinline__ void ln_apply(const uint4& x, const __nv_bfloat16* __restrict__ w,
                                         const __nv_bfloat16* __restrict__ b, int v, float2 stats, float (&o)[8]) {
  float f[8], wv[8], bv[8];
  unpack8(x, f);
  unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
  unpack8(__ldg(reinterpret_cast<const uint4*>(b) + v), bv);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = (f[j] - stats.x) * stats.y * wv[j] + bv[j];
}

// Launch ladder: calls go(VPT, TPR) (std::integral_constant values) for the first VPT of the list whose VPT * TPR
// vectors hold the row's nvec; VLLM_EUNSUPPORTED past the last.  The (VPT, TPR) an entry point picks fixes its
// reduction order, so each keeps its own list.
template <int TPR, int VPT, int... MORE, class Go>
static inline int with_vpt(int nvec, Go&& go) {
  if (nvec <= VPT * TPR) return go(std::integral_constant<int, VPT>{}, std::integral_constant<int, TPR>{});
  if constexpr (sizeof...(MORE) == 0) return VLLM_EUNSUPPORTED;
  else return with_vpt<TPR, MORE...>(nvec, go);
}
