// Vectorised HBM-bound row kernels of the forward hot path (bf16 in/out, fp32 math).
//
//  * RMSNorm  -- replaces apex FusedRMSNorm `cuApplyRMSNorm` (apex/csrc/layer_norm_cuda_kernel.cu:353-437,
//    CPU semantics apex/normalization/fused_layer_norm.py:16-29) == InternRMSNorm
//    (internvit/modeling_intern_vit.py:33-44) == InternLM2RMSNorm (internlm2/modeling_internlm2.py:114-128)
//    == HF LlamaRMSNorm: fp32 sum of squares, x * rsqrt(mean + eps) rounded to the input dtype, THEN times weight.
//    Strided rows so the InternViT q/k norm over the flattened 3200-d slices of the packed qkv tensor
//    (modeling_intern_vit.py:149-153) runs in place with no `torch.stack([q, k, v])` copy.
//  * LayerNorm (CLIP / GDINO nn.LayerNorm): fp32 mean/var, affine.
//  * RoPE, rotate-half form (HF Llama apply_rotary_pos_emb; internlm2/modeling_internlm2.py:218-232):
//    q' = q*cos + rotate_half(q)*sin with cos/sin rounded to bf16 like the reference's cached tables.
//
// One CTA per row; 16-byte loads; the row stays in registers between the reduction and the scaling pass
// (1 read + 1 write of the activation -- the roofline for these ops).
#include "rows.cuh"

namespace {

constexpr int NT = 256;          // threads per CTA

// A row is owned by TPR threads (a warp, 4 warps or the whole CTA); a CTA carries NT/TPR rows.  Each thread keeps
// VPT 16-byte vectors of the row in registers (packed bf16) between the statistics pass and the scaling pass.
// mode 0: RMSNorm (weight only); mode 1: LayerNorm (weight + bias), act 1 applies exact-erf GELU to the normalised row,
// res adds a residual row after it.
template <int MODE, int VPT, int TPR>
__global__ void __launch_bounds__(NT)
norm_rows_kernel(const __nv_bfloat16* x, long long ldx, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ b, __nv_bfloat16* y, long long ldy, long long rows,
                 int cols, float eps, int act, const __nv_bfloat16* __restrict__ res, long long ldr,
                 const int64_t* __restrict__ gidx, long long g_in, long long g_out) {
  __shared__ float sh[NT / 32];
  const int tr = threadIdx.x % TPR;
  const long long row = (long long)blockIdx.x * (NT / TPR) + threadIdx.x / TPR;
  const bool row_ok = row < rows;
  // row gather (Swin window partition): output row (batch, j) normalises input row (batch, gidx[j]); gidx[j] >= g_in marks
  // a padded window slot -> an all-zero output row
  long long src = row;
  bool zero_row = false;
  if (gidx && row_ok) {
    const long long bb = row / g_out;
    const long long si = gidx[row - bb * g_out];
    zero_row = si >= g_in;
    src = bb * g_in + (zero_row ? 0 : si);
  }
  const __nv_bfloat16* xr = x + (row_ok ? src : 0) * ldx;
  __nv_bfloat16* yr = y + (row_ok ? row : 0) * ldy;
  const int nvec = cols / 8;
  uint4 reg[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = tr + i * TPR;
    reg[i] = (v < nvec && row_ok) ? *(reinterpret_cast<const uint4*>(xr) + v) : make_uint4(0, 0, 0, 0);  // may alias y
  }
  float2 st;
  if constexpr (MODE == 1) st = ln_stats<VPT, TPR, NT>(reg, cols, eps, sh);
  else st.y = rms_rstd<VPT, TPR, true, NT>(reg, cols, eps, sh);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = tr + i * TPR;
    if (v < nvec && row_ok) {
      uint4 out;
      if constexpr (MODE == 1) {
        float o[8];
        ln_apply(reg[i], w, b, v, st, o);
        if (act == 1) {                                  // exact-erf GELU on the normalised row (LN -> GELU chains)
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = 0.5f * o[j] * (1.f + erff(o[j] * 0.70710678118654752f));
        }
        if (res) {                                       // y = residual + LN(x): the post-norm residual of InternImage-H
          float rv[8]; unpack8(*(reinterpret_cast<const uint4*>(res + row * ldr) + v), rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rv[j];
        }
        out = pack8(o);
      } else {
        out = rms_apply(reg[i], w, v, st.y);
      }
      *(reinterpret_cast<uint4*>(yr) + v) = zero_row ? make_uint4(0u, 0u, 0u, 0u) : out;
    }
  }
}

template <int MODE>
int launch_norm(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, long long rows,
                int cols, float eps, cudaStream_t st, int act = 0, const void* res = nullptr, long long ldr = 0,
                const int64_t* gidx = nullptr, long long g_in = 0, long long g_out = 0) {
  auto go = [&](auto vpt, auto tpr) -> int {
    constexpr int VPT = decltype(vpt)::value, TPR = decltype(tpr)::value;
    const long long blocks = (rows + NT / TPR - 1) / (NT / TPR);
    if (blocks > 2147483647LL) return VLLM_EUNSUPPORTED;
    norm_rows_kernel<MODE, VPT, TPR><<<(unsigned)blocks, NT, 0, st>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)w, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, ldy, rows,
        cols, eps, act, (const __nv_bfloat16*)res, ldr, gidx, g_in, g_out);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  };
  // a warp per row up to 128 vectors, 4 warps up to 1024, the whole CTA beyond
  const int nvec = cols / 8;
  if (nvec <= 128) return with_vpt<32, 1, 2, 4>(nvec, go);
  if (nvec <= 1024) return with_vpt<128, 2, 4, 8>(nvec, go);
  return with_vpt<256, 8>(nvec, go);
}

// qk [T, heads, 128]-style rows inside a packed tensor: element (t, h, d) at base + t*ld + h*hd + d.
// cos/sin [T, hd] bf16 (already gathered per position).  In place.
__global__ void __launch_bounds__(128)
rope_kernel(__nv_bfloat16* __restrict__ x, long long ld, const __nv_bfloat16* __restrict__ cs,
            const __nv_bfloat16* __restrict__ sn, int heads, int hd, long long tokens) {
  // one warp per (token, head); lane handles hd/64 pairs (d, d + hd/2)
  const long long wid = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= tokens * heads) return;
  const long long t = wid / heads;
  const int h = (int)(wid % heads);
  __nv_bfloat16* p = x + t * ld + (long long)h * hd;
  const __nv_bfloat16* c = cs + t * hd;
  const __nv_bfloat16* s = sn + t * hd;
  const int half = hd / 2;
  for (int d = (threadIdx.x & 31) * 2; d < half; d += 64) {
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(p + d);
    const __nv_bfloat162 bq = *reinterpret_cast<const __nv_bfloat162*>(p + d + half);
    const float2 af = __bfloat1622float2(a), bf = __bfloat1622float2(bq);
    const float2 c0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(c + d));
    const float2 c1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(c + d + half));
    const float2 s0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(s + d));
    const float2 s1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(s + d + half));
    // reference rounds each bf16 product, then the sum: (q*cos) + (rotate_half(q)*sin)
    auto r = [](float v) { return __bfloat162float(__float2bfloat16(v)); };
    float2 lo, hi;
    lo.x = r(af.x * c0.x) + r(-bf.x * s0.x); lo.y = r(af.y * c0.y) + r(-bf.y * s0.y);
    hi.x = r(bf.x * c1.x) + r(af.x * s1.x);  hi.y = r(bf.y * c1.y) + r(af.y * s1.y);
    *reinterpret_cast<__nv_bfloat162*>(p + d) = __floats2bfloat162_rn(lo.x, lo.y);
    *reinterpret_cast<__nv_bfloat162*>(p + d + half) = __floats2bfloat162_rn(hi.x, hi.y);
  }
}

// 16-byte form of the same arithmetic (bit-identical results): a thread owns 8 consecutive d of the low half and the
// 8 partners of the high half of one (token, head); hd/16 threads per head, so a 128-d head is 8 threads x 6 x LDG.128.
__global__ void __launch_bounds__(256)
rope_vec_kernel(__nv_bfloat16* __restrict__ x, long long ld, const __nv_bfloat16* __restrict__ cs,
                const __nv_bfloat16* __restrict__ sn, int heads, int hd, long long tokens) {
  const int tph = hd / 16;                                   // threads per head
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = tokens * heads * tph;
  if (idx >= total) return;
  const int v = (int)(idx % tph);
  const long long th = idx / tph;
  const long long t = th / heads;
  const int h = (int)(th % heads);
  const int half = hd / 2, d = v * 8;
  __nv_bfloat16* p = x + t * ld + (long long)h * hd;
  float a[8], b[8], c0[8], c1[8], s0[8], s1[8], lo[8], hi[8];
  unpack8(*reinterpret_cast<const uint4*>(p + d), a);
  unpack8(*reinterpret_cast<const uint4*>(p + d + half), b);
  unpack8(__ldg(reinterpret_cast<const uint4*>(cs + t * hd + d)), c0);
  unpack8(__ldg(reinterpret_cast<const uint4*>(cs + t * hd + d + half)), c1);
  unpack8(__ldg(reinterpret_cast<const uint4*>(sn + t * hd + d)), s0);
  unpack8(__ldg(reinterpret_cast<const uint4*>(sn + t * hd + d + half)), s1);
  auto r = [](float q) { return __bfloat162float(__float2bfloat16(q)); };
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    lo[j] = r(a[j] * c0[j]) + r(-b[j] * s0[j]);
    hi[j] = r(b[j] * c1[j]) + r(a[j] * s1[j]);
  }
  *reinterpret_cast<uint4*>(p + d) = pack8(lo);
  *reinterpret_cast<uint4*>(p + d + half) = pack8(hi);
}

int check_rows(const void* x, long long ldx, const void* y, long long ldy, long long rows, int cols) {
  if (rows < 0 || cols <= 0) return VLLM_EINVAL;
  if (rows == 0) return 1000;
  if (!x || !y) return VLLM_EINVAL;
  if (cols % 8 || cols > 8 * 256 * 8) return VLLM_EUNSUPPORTED;
  if (ldx % 8 || ldy % 8 || !vllm_aligned(x, 16) || !vllm_aligned(y, 16)) return VLLM_EALIGN;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  return VLLM_OK;
}

}  // namespace

extern "C" {

int vllm_rmsnorm_bf16(const void* x, long long ldx, const void* weight, void* y, long long ldy, long long rows,
                      int cols, float eps, void* stream) {
  int rc = check_rows(x, ldx, y, ldy, rows, cols);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!weight || !vllm_aligned(weight, 16)) return VLLM_EINVAL;
  return launch_norm<0>(x, ldx, weight, nullptr, y, ldy, rows, cols, eps, (cudaStream_t)stream);
}

int vllm_layernorm_bf16(const void* x, long long ldx, const void* weight, const void* bias, void* y, long long ldy,
                        long long rows, int cols, float eps, void* stream) {
  int rc = check_rows(x, ldx, y, ldy, rows, cols);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!weight || !bias || !vllm_aligned(weight, 16) || !vllm_aligned(bias, 16)) return VLLM_EINVAL;
  return launch_norm<1>(x, ldx, weight, bias, y, ldy, rows, cols, eps, (cudaStream_t)stream);
}

int vllm_layernorm_gelu_bf16(const void* x, long long ldx, const void* weight, const void* bias, void* y,
                             long long ldy, long long rows, int cols, float eps, void* stream) {
  int rc = check_rows(x, ldx, y, ldy, rows, cols);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!weight || !bias || !vllm_aligned(weight, 16) || !vllm_aligned(bias, 16)) return VLLM_EINVAL;
  return launch_norm<1>(x, ldx, weight, bias, y, ldy, rows, cols, eps, (cudaStream_t)stream, 1);
}

int vllm_layernorm_gather_bf16(const void* x, long long ldx, const int64_t* index, long long rows_in, long long rows_out,
                               long long batch, const void* weight, const void* bias, void* y, long long ldy, int cols,
                               float eps, void* stream) {
  if (rows_in <= 0 || rows_out < 0 || batch < 0) return VLLM_EINVAL;
  if (!index) return VLLM_EINVAL;
  int rc = check_rows(x, ldx, y, ldy, batch * rows_out, cols);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!weight || !bias || !vllm_aligned(weight, 16) || !vllm_aligned(bias, 16)) return VLLM_EINVAL;
  return launch_norm<1>(x, ldx, weight, bias, y, ldy, batch * rows_out, cols, eps, (cudaStream_t)stream, 0, nullptr, 0, index,
                        rows_in, rows_out);
}

int vllm_layernorm_residual_bf16(const void* x, long long ldx, const void* weight, const void* bias,
                                 const void* residual, long long ldr, void* y, long long ldy, long long rows, int cols,
                                 float eps, void* stream) {
  int rc = check_rows(x, ldx, y, ldy, rows, cols);
  if (rc == 1000) return VLLM_OK;
  if (rc) return rc;
  if (!weight || !bias || !residual || !vllm_aligned(weight, 16) || !vllm_aligned(bias, 16)) return VLLM_EINVAL;
  if (!vllm_aligned(residual, 16) || ldr % 8) return VLLM_EALIGN;
  return launch_norm<1>(x, ldx, weight, bias, y, ldy, rows, cols, eps, (cudaStream_t)stream, 0, residual, ldr);
}

int vllm_rope_bf16(void* x, long long ld, const void* cos, const void* sin, long long tokens, int heads,
                   int head_dim, void* stream) {
  if (tokens < 0 || heads <= 0 || head_dim <= 0) return VLLM_EINVAL;
  if (tokens == 0) return VLLM_OK;
  if (!x || !cos || !sin) return VLLM_EINVAL;
  if (head_dim % 4 || ld % 2) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(x, 4) || !vllm_aligned(cos, 4) || !vllm_aligned(sin, 4)) return VLLM_EALIGN;
  if (head_dim % 16 == 0 && ld % 8 == 0 && vllm_aligned(x, 16) && vllm_aligned(cos, 16) && vllm_aligned(sin, 16)) {
    const long long threads = tokens * heads * (head_dim / 16);
    const long long vblocks = (threads + 255) / 256;
    if (vblocks > 2147483647LL) return VLLM_EUNSUPPORTED;
    rope_vec_kernel<<<(unsigned)vblocks, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)x, ld, (const __nv_bfloat16*)cos,
                                                                        (const __nv_bfloat16*)sin, heads, head_dim, tokens);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  }
  const long long warps = tokens * heads;
  const long long blocks = (warps + 3) / 4;
  if (blocks > 2147483647LL) return VLLM_EUNSUPPORTED;
  rope_kernel<<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)x, ld, (const __nv_bfloat16*)cos,
                                                                 (const __nv_bfloat16*)sin, heads, head_dim, tokens);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // extern "C"
