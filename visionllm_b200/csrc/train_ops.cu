// Row kernels of the training-side path of the LLM decoder (BASELINE cfg 5 "fwd+bwd step"): the backward of the
// HBM-bound forward ops of fused_ops.cu / the GEMM epilogues, and the loss.  bf16 activations / gradients, fp32 math.
//
//   rmsnorm_bwd_kernel     autograd of HF LlamaRMSNorm == InternLM2RMSNorm (internlm2/modeling_internlm2.py:114-128) ==
//                          apex rms_backward_affine (apex/csrc/layer_norm_cuda_kernel.cu cuComputeGradInput / GradGammaBeta):
//                          n = x * rsqrt(mean(x^2) + eps); y = w * n;  dn = dy * w;
//                          dx = rstd * (dn - n * mean(dn * n));  dw += sum_rows dy * n
//   swiglu_fwd / bwd       h = silu(g) * u on the interleaved (gate, up) columns the gate|up GEMM produces
//                          (LlamaMLP / InternLM2MLP: down(act(gate(x)) * up(x))); dg = dh * u * silu'(g), du = dh * silu(g)
//   softmax_causal_kernel  P = softmax(scale * S) over keys <= query (fp32 softmax like HF eager attention), zeros above
//                          the diagonal; attn_ds_kernel: dS = scale * P * (dP - sum_k dP * P)  (softmax backward), zeros above
//   ce_loss_kernel         visionllmv2/model/modeling_visionllmv2.py:741-757: CrossEntropyLoss (mean over labels != -100) of
//                          fp32 logits rows vs int64 labels; writes the loss sum and dlogits = (softmax - onehot) / n_valid.
#include "rows.cuh"
#include "msda_common.cuh"

namespace {

// A CTA (256 threads) owns rows_per_cta consecutive rows; VPT 16-byte vectors per thread stay in registers.  Its dw
// contribution (fp32, summed over its rows) goes to row blockIdx.x of partials [gridDim.x, cols].
template <int VPT>
__global__ void __launch_bounds__(256)
rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ w,
                   const __nv_bfloat16* __restrict__ dy, long long ldy, __nv_bfloat16* __restrict__ dx, long long lddx,
                   long long rows, int cols, float eps, int rows_per_cta, float* __restrict__ partials) {
  __shared__ float sh[8];
  const int nvec = cols / 8;
  float dwacc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  for (long long row = r0; row < r0 + rows_per_cta && row < rows; ++row) {
    uint4 xr[VPT], gr[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * 256;
      xr[i] = gr[i] = make_uint4(0u, 0u, 0u, 0u);
      if (v < nvec) {
        xr[i] = *(reinterpret_cast<const uint4*>(x + row * ldx) + v);
        gr[i] = *(reinterpret_cast<const uint4*>(dy + row * ldy) + v);
      }
    }
    const float rstd = rms_rstd<VPT, 256>(xr, cols, eps, sh);
    float dot = 0.f;                                        // sum dn * n
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * 256;
      if (v < nvec) {
        float f[8], g[8], wv[8];
        unpack8(xr[i], f); unpack8(gr[i], g); unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float n = f[j] * rstd;
          dot += g[j] * wv[j] * n;
          // dw uses the forward's bf16-rounded normalised value (y = w * bf16(n)), like autograd through the cast
          dwacc[i][j] += g[j] * __bfloat162float(__float2bfloat16(n));
        }
      }
    }
    const float mdot = row_sum<256>(dot, sh) / cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * 256;
      if (v < nvec) {
        float f[8], g[8], wv[8], o[8];
        unpack8(xr[i], f); unpack8(gr[i], g); unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * wv[j] - f[j] * rstd * mdot);
        *(reinterpret_cast<uint4*>(dx + row * lddx) + v) = pack8(o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * 256;
    if (v < nvec) {                                        // one coalesced row of partials per CTA, summed by the second kernel
      float* pr = partials + (size_t)blockIdx.x * cols + v * 8;
      *reinterpret_cast<float4*>(pr) = make_float4(dwacc[i][0], dwacc[i][1], dwacc[i][2], dwacc[i][3]);
      *reinterpret_cast<float4*>(pr + 4) = make_float4(dwacc[i][4], dwacc[i][5], dwacc[i][6], dwacc[i][7]);
    }
  }
}

// dw[c] = sum over the n per-CTA partial rows in a fixed order (deterministic): a CTA owns 32 columns,
// its 8 warps take every 8th row (128-byte coalesced reads), shared-memory tree at the end
__global__ void __launch_bounds__(256)
colsum_partials_kernel(const float* __restrict__ partials, float* __restrict__ dw, int n, int cols) {
  __shared__ float sh[8][32];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float a = 0.f;
  if (c < cols)
    for (int r = grp; r < n; r += 8) a += partials[(size_t)r * cols + c];
  sh[grp][lane] = a;
  __syncthreads();
  if (grp == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) t += sh[g][lane];
    dw[c] = t;
  }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// gu [rows, 2I] interleaved (g0, u0, g1, u1, ...) -> h [rows, I]; 8 outputs per thread
__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gu, long long ldgu, __nv_bfloat16* __restrict__ h, long long ldh,
                  long long rows, int inter) {
  const int vec_per_row = inter / 8;
  const long long total = rows * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vec_per_row;
    const int v = (int)(i - row * vec_per_row);
    const uint4* src = reinterpret_cast<const uint4*>(gu + row * ldgu) + 2 * v;
    float a[8], b[8], o[8];
    unpack8(src[0], a); unpack8(src[1], b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[j] = a[2 * j] * sigmoidf_(a[2 * j]) * a[2 * j + 1];
      o[4 + j] = b[2 * j] * sigmoidf_(b[2 * j]) * b[2 * j + 1];
    }
    *(reinterpret_cast<uint4*>(h + row * ldh) + v) = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ gu, long long ldgu, const __nv_bfloat16* __restrict__ dh, long long lddh,
                  __nv_bfloat16* __restrict__ dgu, long long lddgu, long long rows, int inter) {
  const int vec_per_row = inter / 8;
  const long long total = rows * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vec_per_row;
    const int v = (int)(i - row * vec_per_row);
    const uint4* src = reinterpret_cast<const uint4*>(gu + row * ldgu) + 2 * v;
    float a[8], b[8], d[8], oa[8], ob[8];
    unpack8(src[0], a); unpack8(src[1], b);
    unpack8(*(reinterpret_cast<const uint4*>(dh + row * lddh) + v), d);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      {
        const float g = a[2 * j], u = a[2 * j + 1], s = sigmoidf_(g);
        oa[2 * j] = d[j] * u * s * (1.f + g * (1.f - s));
        oa[2 * j + 1] = d[j] * g * s;
      }
      {
        const float g = b[2 * j], u = b[2 * j + 1], s = sigmoidf_(g);
        ob[2 * j] = d[4 + j] * u * s * (1.f + g * (1.f - s));
        ob[2 * j + 1] = d[4 + j] * g * s;
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(dgu + row * lddgu) + 2 * v;
    dst[0] = pack8(oa); dst[1] = pack8(ob);
  }
}

// S [n_mat, T, T] bf16 (row pitch lds, matrix pitch T*lds) -> P in place: softmax over keys j <= i of scale * S, zeros for j > i.
// With `lens` (key lengths, one per batch row of heads_per_batch consecutive matrices) the keys are j <= i and j < len:
// P = 0 for j >= len, and S is not used there (a NaN in a masked key cannot leak); a row with no key is all zeros.
// One CTA per row; T <= 256 * 8 * VPT.
template <int VPT>
__global__ void __launch_bounds__(256)
softmax_causal_kernel(__nv_bfloat16* __restrict__ s, long long lds, int T, float scale, const int* __restrict__ lens,
                      int heads_per_batch) {
  __shared__ float sh[8];
  const long long row_g = blockIdx.x;                        // matrix * T + i
  const int i = (int)(row_g % T);
  const int last = lens ? min(i, lens[row_g / T / heads_per_batch] - 1) : i;   // last visible key
  __nv_bfloat16* sr = s + row_g * lds;
  const int nvec = T / 8;
  float v[VPT][8];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = threadIdx.x + k * 256;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[k][j] = -INFINITY;
    if (vi < nvec && vi * 8 <= last) {
      float f[8]; unpack8(*(reinterpret_cast<const uint4*>(sr) + vi), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) if (vi * 8 + j <= last) { v[k][j] = f[j] * scale; mx = fmaxf(mx, v[k][j]); }
    }
  }
  mx = row_max<256>(mx, sh);
  if (lens && mx == -INFINITY) mx = 0.f;                     // no visible key (length 0): exp(-inf) = 0 everywhere
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < VPT; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[k][j] = __expf(v[k][j] - mx); sum += v[k][j]; }     // exp(-inf) = 0 above the diagonal
  sum = row_sum<256>(sum, sh);
  const float inv = lens && !(sum > 0.f) ? 0.f : 1.f / sum;  // without lengths: the original arithmetic for any input
  // zeros are only needed inside the 256-aligned diagonal block: the causal batched GEMMs (gemm.cu, causal 2 / 3) never read
  // a 64-column k-block that lies wholly above a tile's diagonal block, and tiles are at most 256 rows
  const int wvec = min(nvec, ((i >> 8) + 1) * 32);
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = threadIdx.x + k * 256;
    if (vi < wvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = v[k][j] * inv;
      *(reinterpret_cast<uint4*>(sr) + vi) = pack8(o);
    }
  }
}

// dP [.., T, T] -> dS in place: dS = scale * P * (dP - sum_j dP_j P_j); zeros above the diagonal (P is zero there)
template <int VPT>
__global__ void __launch_bounds__(256)
attn_ds_kernel(const __nv_bfloat16* __restrict__ p, __nv_bfloat16* __restrict__ dp, long long ld, int T, float scale) {
  __shared__ float sh[8];
  const long long row_g = blockIdx.x;
  const int i = (int)(row_g % T);
  const __nv_bfloat16* pr = p + row_g * ld;
  __nv_bfloat16* dr = dp + row_g * ld;
  const int nvec = T / 8;
  float pv[VPT][8], dv[VPT][8];
  float dot = 0.f;
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = threadIdx.x + k * 256;
#pragma unroll
    for (int j = 0; j < 8; ++j) { pv[k][j] = 0.f; dv[k][j] = 0.f; }
    if (vi < nvec && vi * 8 <= i) {
      unpack8(*(reinterpret_cast<const uint4*>(pr) + vi), pv[k]);
      unpack8(*(reinterpret_cast<const uint4*>(dr) + vi), dv[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (vi * 8 + j > i) { pv[k][j] = 0.f; dv[k][j] = 0.f; }       // dP above the diagonal may be uncomputed garbage
        dot += pv[k][j] * dv[k][j];
      }
    }
  }
  dot = row_sum<256>(dot, sh);
  const int wvec = min(nvec, ((i >> 8) + 1) * 32);            // see softmax_causal_kernel
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = threadIdx.x + k * 256;
    if (vi < wvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = scale * pv[k][j] * (dv[k][j] - dot);
      *(reinterpret_cast<uint4*>(dr) + vi) = pack8(o);
    }
  }
}

// [B, T, 3, H, D] (the packed q | k | v projection rows) <-> [3, B, H, T, D] (every (batch, head) matrix of q, k, v stacked
// along rows for the block-diagonal batched GEMMs of the attention backward), 16-byte vectors; `to_stacked` = 0 goes back
// (the packed gradient).  NP = 3 for qkv, 1 for a plain [B, T, H, D] tensor (dO).
__global__ void __launch_bounds__(256)
head_stack_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B, int T, int NP, int H, int DV,
                  int to_stacked, long long n_vec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    // i indexes the STACKED tensor [NP, B, H, T, DV] (coalesced on the stacked side, 256-byte runs on the packed side)
    const int d = (int)(i % DV);
    long long r = i / DV;
    const int t = (int)(r % T); r /= T;
    const int h = (int)(r % H); r /= H;
    const int b = (int)(r % B);
    const int part = (int)(r / B);
    const long long packed = ((((long long)b * T + t) * NP + part) * H + h) * DV + d;
    if (to_stacked) dst[i] = src[packed];
    else dst[packed] = src[i];
  }
}

// Grouped-query form of the same layout change: packed projection rows [B, T, (nq + 2 nkv) D] with row pitch ld_vec
// 16-byte vectors (q heads, then k heads, then v heads) <-> three stacks Q [B, nq, TP, D], K [B, nkv, TP, D], V [B, nkv, TP, D].
// i indexes the concatenation Q | K | V of the stacks (coalesced on the stacked side); the pitch gap of a packed row is
// neither read nor written.  Stack rows t >= T (TP > T pads every matrix) are written as zeros going to the stacks and
// skipped coming back.  NKV = 0 stacks the q heads alone.
__global__ void __launch_bounds__(256)
head_stack_qkv_kernel(uint4* __restrict__ packed, long long ld_vec, uint4* __restrict__ q, uint4* __restrict__ k,
                      uint4* __restrict__ v, int B, int T, int TP, int NQ, int NKV, int DV, int to_stacked, long long n_vec) {
  const long long n_q = (long long)B * NQ * TP * DV, n_kv = (long long)B * NKV * TP * DV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    uint4* st = q; int heads = NQ, h0 = 0;
    if (r >= n_q) {
      r -= n_q;
      if (r < n_kv) { st = k; heads = NKV; h0 = NQ; }
      else { r -= n_kv; st = v; heads = NKV; h0 = NQ + NKV; }
    }
    const long long si = r;
    const int d = (int)(r % DV); r /= DV;
    const int t = (int)(r % TP); r /= TP;
    const int h = (int)(r % heads);
    const int b = (int)(r / heads);
    if (t >= T) {
      if (to_stacked) st[si] = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const long long pi = ((long long)b * T + t) * ld_vec + (long long)(h0 + h) * DV + d;
    if (to_stacked) st[si] = packed[pi];
    else packed[pi] = st[si];
  }
}

// logits fp32 [rows, V] (pitch ld), labels int64 [rows] (-100 = ignore), n_valid: device int64 scalar.
// loss_sum += -log softmax(logits)[label] (fp32 atomic); dlogits bf16 [rows, V] (pitch ldd) = (softmax - onehot) / n_valid,
// zero rows for ignored labels.  One CTA (512 threads) per row, three passes over the row (max, sum, write).
__global__ void __launch_bounds__(512)
ce_loss_kernel(const float* __restrict__ logits, long long ld, const int64_t* __restrict__ labels,
               const int64_t* __restrict__ n_valid, int V, float* __restrict__ loss_sum, __nv_bfloat16* __restrict__ dlogits,
               long long ldd) {
  __shared__ float sh[16];
  const long long row = blockIdx.x;
  const float* lr = logits + row * ld;
  const long long label = labels[row];
  __nv_bfloat16* dr = dlogits ? dlogits + row * ldd : nullptr;
  if (label < 0 || label >= V) {                             // IGNORE_INDEX (-100): no loss, zero gradient
    if (dr) for (int c = threadIdx.x; c < V; c += 512) dr[c] = __float2bfloat16(0.f);
    return;
  }
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += 512) mx = fmaxf(mx, lr[c]);
  mx = row_max<512>(mx, sh);
  float sum = 0.f;
  for (int c = threadIdx.x; c < V; c += 512) sum += expf(lr[c] - mx);
  sum = row_sum<512>(sum, sh);
  const float lse = mx + logf(sum);
  if (threadIdx.x == 0) atomicAdd(loss_sum, lse - lr[label]);
  if (dr) {
    const float invn = 1.f / (float)(*n_valid);
    for (int c = threadIdx.x; c < V; c += 512) {
      float g = expf(lr[c] - lse);
      if (c == label) g -= 1.f;
      dr[c] = __float2bfloat16(g * invn);
    }
  }
}

// x [rows, cols] bf16 (pitch ld) *= *scale in place: fp32 product, one rounding; the scale is read on the device (the
// upstream gradient of a loss, so no host sync).  One CTA per row, 16-byte vectors, the cols % 8 tail scalar.
__global__ void __launch_bounds__(256)
scale_rows_kernel(__nv_bfloat16* __restrict__ x, long long ld, int cols, const float* __restrict__ scale) {
  const float s = *scale;
  __nv_bfloat16* xr = x + (long long)blockIdx.x * ld;
  const int nvec = cols / 8;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    uint4* p = reinterpret_cast<uint4*>(xr) + v;
    float f[8]; unpack8(*p, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= s;
    *p = pack8(f);
  }
  for (int c = nvec * 8 + threadIdx.x; c < cols; c += 256) xr[c] = __float2bfloat16(__bfloat162float(xr[c]) * s);
}

// ---- backward of the vision-language bridge and of the sequence assembly (the multimodal training step) ----

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// d/du of 0.5 u (1 + erf(u / sqrt 2)) = Phi(u) + u phi(u)
__device__ __forceinline__ float gelu_erf_grad(float u) {
  return 0.5f * (1.f + erff(u * 0.70710678118654752f)) + u * 0.39894228040143268f * expf(-0.5f * u * u);
}

// y = gelu(u) (BACKWARD = 0) or dx = dy * gelu'(u) (BACKWARD = 1) on [rows, cols] bf16, 8 elements per thread
template <bool BACKWARD>
__global__ void __launch_bounds__(256)
gelu_kernel(const __nv_bfloat16* __restrict__ u, long long ldu, const __nv_bfloat16* __restrict__ dy, long long lddy,
            __nv_bfloat16* __restrict__ out, long long ldo, long long rows, int cols) {
  const int vec_per_row = cols / 8;
  const long long total = rows * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vec_per_row;
    const int v = (int)(i - row * vec_per_row);
    float a[8], o[8];
    unpack8(*(reinterpret_cast<const uint4*>(u + row * ldu) + v), a);
    if constexpr (BACKWARD) {
      float g[8];
      unpack8(*(reinterpret_cast<const uint4*>(dy + row * lddy) + v), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j] * gelu_erf_grad(a[j]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = gelu_erf(a[j]);
    }
    *(reinterpret_cast<uint4*>(out + row * ldo) + v) = pack8(o);
  }
}

// Column sums of dy [rows, cols] over the rows of a CTA, in row order: CTA (x, y) owns rows [x rpc, (x + 1) rpc) and the
// 256 16-byte column vectors of block y; its sums go to row x of partials [gridDim.x, cols] (then colsum_partials_kernel).
__global__ void __launch_bounds__(256)
colsum_rows_kernel(const __nv_bfloat16* __restrict__ dy, long long ldy, long long rows, int cols, int rows_per_cta,
                   float* __restrict__ partials) {
  const int v = blockIdx.y * 256 + threadIdx.x;
  if (v >= cols / 8) return;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  for (long long row = r0; row < r0 + rows_per_cta && row < rows; ++row) {
    float g[8];
    unpack8(*(reinterpret_cast<const uint4*>(dy + row * ldy) + v), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += g[j];
  }
  float* pr = partials + (size_t)blockIdx.x * cols + v * 8;
  *reinterpret_cast<float4*>(pr) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  *reinterpret_cast<float4*>(pr + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// nn.LayerNorm weight / bias gradients: xhat = (x - mean) * rstd (fp32, the forward's statistics recomputed by ln_stats);
// dgamma += dy * xhat, dbeta += dy over the CTA's rows in order -> rows x (dgamma) and n + x (dbeta) of partials [2n, cols].
template <int VPT>
__global__ void __launch_bounds__(256)
layernorm_bwd_wb_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ dy,
                        long long ldy, long long rows, int cols, float eps, int rows_per_cta, float* __restrict__ partials) {
  __shared__ float sh[8];
  const int nvec = cols / 8;
  float gacc[VPT][8], bacc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) gacc[i][j] = bacc[i][j] = 0.f;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  for (long long row = r0; row < r0 + rows_per_cta && row < rows; ++row) {
    uint4 xr[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * 256;
      xr[i] = v < nvec ? *(reinterpret_cast<const uint4*>(x + row * ldx) + v) : make_uint4(0u, 0u, 0u, 0u);
    }
    const float2 st = ln_stats<VPT, 256>(xr, cols, eps, sh);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * 256;
      if (v < nvec) {
        float f[8], g[8];
        unpack8(xr[i], f); unpack8(*(reinterpret_cast<const uint4*>(dy + row * ldy) + v), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) { gacc[i][j] += g[j] * ((f[j] - st.x) * st.y); bacc[i][j] += g[j]; }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * 256;
    if (v < nvec) {
      float* pg = partials + (size_t)blockIdx.x * cols + v * 8;
      float* pb = partials + (size_t)(gridDim.x + blockIdx.x) * cols + v * 8;
      *reinterpret_cast<float4*>(pg) = make_float4(gacc[i][0], gacc[i][1], gacc[i][2], gacc[i][3]);
      *reinterpret_cast<float4*>(pg + 4) = make_float4(gacc[i][4], gacc[i][5], gacc[i][6], gacc[i][7]);
      *reinterpret_cast<float4*>(pb) = make_float4(bacc[i][0], bacc[i][1], bacc[i][2], bacc[i][3]);
      *reinterpret_cast<float4*>(pb + 4) = make_float4(bacc[i][4], bacc[i][5], bacc[i][6], bacc[i][7]);
    }
  }
}

// Backward of vllm_layernorm_gelu_bf16 (y = gelu(z), z = n w + b, n = (x - mean) rstd; the region encoder's LayerNorm2d ->
// GELU): the statistics are recomputed by ln_stats at the forward's (VPT, TPR), z by ln_apply, so both are the forward's
// bits.  g = dy gelu'(z);  dx = rstd (w g - mean(w g) - n mean(w g n)), one rounding;  dweight += g n, dbias += g.
// A row is owned by TPR threads, a CTA holds 256 / TPR row slots; slot s owns rows [s rps, (s + 1) rps) in order and
// writes its sums to rows s (dweight) and n_slots + s (dbias) of partials [2 n_slots, cols] (colsum_partials_kernel).
// Every slot of a CTA runs rps iterations (the row reductions of TPR > 32 synchronise the CTA); a row past the end is
// zeros and neither stored nor summed.
template <int VPT, int TPR>
__global__ void __launch_bounds__(256)
layernorm_gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ w,
                          const __nv_bfloat16* __restrict__ b, const __nv_bfloat16* __restrict__ dy, long long ldy,
                          __nv_bfloat16* __restrict__ dx, long long lddx, long long rows, int cols, float eps, int rps,
                          long long n_slots, float* __restrict__ partials) {
  __shared__ float sh[8];
  const int tr = threadIdx.x % TPR, nvec = cols / 8;
  const long long slot = (long long)blockIdx.x * (256 / TPR) + threadIdx.x / TPR;
  const bool slot_ok = slot < n_slots;
  float gacc[VPT][8], bacc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) gacc[i][j] = bacc[i][j] = 0.f;
  for (int k = 0; k < rps; ++k) {
    const long long row = slot * rps + k;
    const bool ok = slot_ok && row < rows;
    uint4 xr[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = tr + i * TPR;
      xr[i] = (ok && v < nvec) ? *(reinterpret_cast<const uint4*>(x + row * ldx) + v) : make_uint4(0u, 0u, 0u, 0u);
    }
    const float2 st = ln_stats<VPT, TPR, 256>(xr, cols, eps, sh);
    float s1 = 0.f, s2 = 0.f;                                 // sum w g, sum w g n
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = tr + i * TPR;
      if (ok && v < nvec) {
        float f[8], z[8], g[8], wv[8];
        unpack8(xr[i], f); unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
        unpack8(*(reinterpret_cast<const uint4*>(dy + row * ldy) + v), g);
        ln_apply(xr[i], w, b, v, st, z);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float n = (f[j] - st.x) * st.y;
          g[j] *= gelu_erf_grad(z[j]);
          gacc[i][j] += g[j] * n;
          bacc[i][j] += g[j];
          s1 += wv[j] * g[j];
          s2 += wv[j] * g[j] * n;
        }
      }
    }
    const float m1 = row_sum<TPR, true, 256>(s1, sh) / cols;
    const float m2 = row_sum<TPR, true, 256>(s2, sh) / cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = tr + i * TPR;
      if (ok && v < nvec) {
        float f[8], z[8], g[8], wv[8], o[8];
        unpack8(xr[i], f); unpack8(__ldg(reinterpret_cast<const uint4*>(w) + v), wv);
        unpack8(*(reinterpret_cast<const uint4*>(dy + row * ldy) + v), g);
        ln_apply(xr[i], w, b, v, st, z);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float n = (f[j] - st.x) * st.y;
          o[j] = st.y * (wv[j] * (g[j] * gelu_erf_grad(z[j])) - m1 - n * m2);
        }
        *(reinterpret_cast<uint4*>(dx + row * lddx) + v) = pack8(o);
      }
    }
  }
  if (!slot_ok) return;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = tr + i * TPR;
    if (v < nvec) {
      float* pg = partials + (size_t)slot * cols + v * 8;
      float* pb = partials + (size_t)(n_slots + slot) * cols + v * 8;
      *reinterpret_cast<float4*>(pg) = make_float4(gacc[i][0], gacc[i][1], gacc[i][2], gacc[i][3]);
      *reinterpret_cast<float4*>(pg + 4) = make_float4(gacc[i][4], gacc[i][5], gacc[i][6], gacc[i][7]);
      *reinterpret_cast<float4*>(pb) = make_float4(bacc[i][0], bacc[i][1], bacc[i][2], bacc[i][3]);
      *reinterpret_cast<float4*>(pb + 4) = make_float4(bacc[i][4], bacc[i][5], bacc[i][6], bacc[i][7]);
    }
  }
}

// Backward of the region encoder's point pooling (the MSDA kernel with one level, point weights pw, then a sum over the
// points and a division by their count).  Splat density of (level l, region r): a[l, r, pixel] = sum over the points in
// index order of pw * (bilinear corner weight of the point at that pixel), fp32, the corner geometry of msda_geom (the
// forward's sampling rule; corners outside the map take nothing).  One thread per pixel, the points staged 256 at a time
// in shared memory: a gather, so the sum has one order and no atomics.
__global__ void __launch_bounds__(256)
point_density_kernel(const float* __restrict__ loc, const float* __restrict__ pw, int n_pts, int R, int H, int W,
                     float* __restrict__ density) {
  __shared__ int s_hl[256], s_wl[256];
  __shared__ float s_lh[256], s_lw[256], s_pw[256];
  const int r = blockIdx.y, l = blockIdx.z;
  const int p = blockIdx.x * 256 + threadIdx.x;
  const int py = p / W, px = p - (p / W) * W;
  const long long base = ((long long)l * R + r) * n_pts;
  float a = 0.f;
  for (int c0 = 0; c0 < n_pts; c0 += 256) {
    const int i = c0 + threadIdx.x;
    __syncthreads();
    if (i < n_pts) {
      const float2 xy = *reinterpret_cast<const float2*>(loc + 2 * (base + i));
      const MsdaGeom<float> g = msda_geom<float>(xy.x, xy.y, H, W);
      const bool in = g.mask & 1;
      s_hl[threadIdx.x] = in ? g.h_low : INT_MIN / 2;          // a sample outside the map touches no pixel
      s_wl[threadIdx.x] = g.w_low;
      s_lh[threadIdx.x] = g.lh; s_lw[threadIdx.x] = g.lw;
      s_pw[threadIdx.x] = pw[base + i];
    }
    __syncthreads();
    const int n = min(256, n_pts - c0);
    for (int j = 0; j < n; ++j) {
      const int dh = py - s_hl[j], dw = px - s_wl[j];
      if ((unsigned)dh <= 1u && (unsigned)dw <= 1u) {
        const float wh = dh ? s_lh[j] : msda_sub(1.f, s_lh[j]);
        const float ww = dw ? s_lw[j] : msda_sub(1.f, s_lw[j]);
        a = msda_add(a, msda_mul(s_pw[j], msda_mul(wh, ww)));
      }
    }
  }
  if (p < H * W) density[((long long)l * R + r) * H * W + p] = a;
}

// d_map [R, HW, C] = sum over levels l in order of a[l, r, pixel] * (g[l, r, c] / cnt[l, r]), fp32, one bf16 rounding;
// a level whose count is 0 adds nothing (the forward's 0 / 0 is zeroed by nan_to_num).  8 channels per thread.
__global__ void __launch_bounds__(256)
point_pool_outer_kernel(const float* __restrict__ density, const float* __restrict__ cnt, const __nv_bfloat16* __restrict__ grad,
                        int L, int R, long long HW, int C, __nv_bfloat16* __restrict__ out) {
  const int nvec = C / 8;
  const long long total = (long long)R * HW * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const long long rp = i / nvec;                            // r * HW + pixel
    const int r = (int)(rp / HW);
    const long long p = rp - (long long)r * HW;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int l = 0; l < L; ++l) {
      const float c = cnt[(long long)l * R + r];
      if (c == 0.f) continue;
      const float a = density[((long long)l * R + r) * HW + p];
      float g[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(grad + ((long long)l * R + r) * C) + v), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = msda_add(acc[j], msda_mul(a, __fdiv_rn(g[j], c)));
    }
    *(reinterpret_cast<uint4*>(out + rp * C) + v) = pack8(acc);
  }
}

// Segment sums of the assembly backward: positions sorted stably by destination row (dest[s], ascending, with order[s] the
// position) -> every row r < n_rows of d_src = sum over the positions with destination r of dy[position], fp32 in
// position order, one bf16 rounding; a row no position names is exact 0.  One CTA per destination row.
__global__ void __launch_bounds__(256)
segment_sum_rows_kernel(const int* __restrict__ dest, const int* __restrict__ order, long long n,
                        const __nv_bfloat16* __restrict__ dy, int C, __nv_bfloat16* __restrict__ out, long long n_rows) {
  const int nvec = C / 8;
  for (long long r = blockIdx.x; r < n_rows; r += gridDim.x) {
    long long lo = 0, hi = n;                                 // first s with dest[s] >= r
    while (lo < hi) { const long long mid = (lo + hi) >> 1; if (dest[mid] < r) lo = mid + 1; else hi = mid; }
    for (int v = threadIdx.x; v < nvec; v += 256) {
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      for (long long s = lo; s < n && dest[s] == r; ++s) {
        float g[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(dy + (long long)order[s] * C) + v), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += g[j];
      }
      *(reinterpret_cast<uint4*>(out + r * C) + v) = pack8(acc);
    }
  }
}

}  // namespace

extern "C" {

static int rmsnorm_bwd_ctas(long long rows) {
  const int rows_per_cta = (int)((rows + (long long)vllm_num_sms() * 8 - 1) / ((long long)vllm_num_sms() * 8));
  return rows_per_cta > 0 ? (int)((rows + rows_per_cta - 1) / rows_per_cta) : 0;
}

/* rows of the `partials` workspace vllm_rmsnorm_bwd_ws_bf16 needs for `rows` activation rows */
int vllm_rmsnorm_bwd_partials(long long rows) { return rows > 0 ? rmsnorm_bwd_ctas(rows) : 0; }

int vllm_rmsnorm_bwd_ws_bf16(const void* x, long long ldx, const void* weight, const void* dy, long long ldy, void* dx,
                             long long lddx, float* dweight, float* partials, int n_partials, long long rows, int cols,
                             float eps, void* stream) {
  if (rows < 0 || cols <= 0 || cols % 8) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!x || !weight || !dy || !dx || !dweight || !partials) return VLLM_EINVAL;
  if (ldx % 8 || ldy % 8 || lddx % 8 || !vllm_aligned(x, 16) || !vllm_aligned(dy, 16) || !vllm_aligned(dx, 16) ||
      !vllm_aligned(partials, 16))
    return VLLM_EALIGN;
  const int rows_per_cta = (int)((rows + (long long)vllm_num_sms() * 8 - 1) / ((long long)vllm_num_sms() * 8));
  const int blocks = rmsnorm_bwd_ctas(rows);
  if (n_partials < blocks) return VLLM_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  return with_vpt<256, 1, 2, 4>(cols / 8, [&](auto vpt, auto) {
    rmsnorm_bwd_kernel<decltype(vpt)::value><<<(unsigned)blocks, 256, 0, st>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)weight, (const __nv_bfloat16*)dy, ldy, (__nv_bfloat16*)dx, lddx,
        rows, cols, eps, rows_per_cta, partials);
    VLLM_CHECK_LAUNCH();
    colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials, dweight, blocks, cols);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

int vllm_head_stack_bf16(const void* src, void* dst, int batch, int tokens, int parts, int heads, int head_dim,
                         int to_stacked, void* stream) {
  if (batch < 0 || tokens < 0 || parts <= 0 || heads <= 0 || head_dim <= 0) return VLLM_EINVAL;
  const long long n_vec = (long long)batch * tokens * parts * heads * (head_dim / 8);
  if (n_vec == 0) return VLLM_OK;
  if (!src || !dst) return VLLM_EINVAL;
  if (head_dim % 8) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(src, 16) || !vllm_aligned(dst, 16)) return VLLM_EALIGN;
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  head_stack_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const uint4*)src, (uint4*)dst, batch, tokens, parts,
                                                                       heads, head_dim / 8, to_stacked ? 1 : 0, n_vec);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_head_stack_qkv_bf16(void* packed, long long ld, void* q, void* k, void* v, int batch, int tokens, int nq, int nkv,
                             int head_dim, int to_stacked, void* stream) {
  if (batch < 0 || tokens < 0 || nq <= 0 || nkv <= 0 || head_dim <= 0 || nq % nkv) return VLLM_EINVAL;
  if (ld < (long long)(nq + 2 * nkv) * head_dim) return VLLM_EINVAL;
  if ((long long)batch * tokens == 0) return VLLM_OK;
  if (!packed || !q || !k || !v) return VLLM_EINVAL;
  if (head_dim % 8) return VLLM_EUNSUPPORTED;                 // before n_vec: head_dim < 8 would give no vectors at all
  const long long n_vec = (long long)batch * tokens * (nq + 2 * nkv) * (head_dim / 8);
  if (ld % 8 || !vllm_aligned(packed, 16) || !vllm_aligned(q, 16) || !vllm_aligned(k, 16) || !vllm_aligned(v, 16))
    return VLLM_EALIGN;
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  head_stack_qkv_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((uint4*)packed, ld / 8, (uint4*)q, (uint4*)k,
                                                                           (uint4*)v, batch, tokens, tokens, nq, nkv, head_dim / 8,
                                                                           to_stacked ? 1 : 0, n_vec);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_swiglu_fwd_bf16(const void* gate_up, long long ldgu, void* h, long long ldh, long long rows, int inter, void* stream) {
  if (rows < 0 || inter <= 0 || inter % 8) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!gate_up || !h) return VLLM_EINVAL;
  if (ldgu % 8 || ldh % 8 || !vllm_aligned(gate_up, 16) || !vllm_aligned(h, 16)) return VLLM_EALIGN;
  long long blocks = (rows * (inter / 8) + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  swiglu_fwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)gate_up, ldgu, (__nv_bfloat16*)h, ldh,
                                                                        rows, inter);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_swiglu_bwd_bf16(const void* gate_up, long long ldgu, const void* dh, long long lddh, void* dgate_up, long long lddgu,
                         long long rows, int inter, void* stream) {
  if (rows < 0 || inter <= 0 || inter % 8) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!gate_up || !dh || !dgate_up) return VLLM_EINVAL;
  if (ldgu % 8 || lddh % 8 || lddgu % 8 || !vllm_aligned(gate_up, 16) || !vllm_aligned(dh, 16) || !vllm_aligned(dgate_up, 16))
    return VLLM_EALIGN;
  long long blocks = (rows * (inter / 8) + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  swiglu_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)gate_up, ldgu,
                                                                        (const __nv_bfloat16*)dh, lddh, (__nv_bfloat16*)dgate_up,
                                                                        lddgu, rows, inter);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_softmax_causal_bf16(void* s, long long ld, long long n_mat, int T, float scale, void* stream) {
  if (n_mat < 0 || T <= 0 || T % 8 || ld < T || ld % 8) return VLLM_EINVAL;
  if (n_mat == 0) return VLLM_OK;
  if (!s) return VLLM_EINVAL;
  if (!vllm_aligned(s, 16)) return VLLM_EALIGN;
  const long long rows = n_mat * T;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  return with_vpt<256, 1, 2, 4>(T / 8, [&](auto vpt, auto) {
    softmax_causal_kernel<decltype(vpt)::value><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)s, ld, T, scale,
                                                                                                nullptr, 1);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

int vllm_attn_ds_bf16(const void* p, void* dp, long long ld, long long n_mat, int T, float scale, void* stream) {
  if (n_mat < 0 || T <= 0 || T % 8 || ld < T || ld % 8) return VLLM_EINVAL;
  if (n_mat == 0) return VLLM_OK;
  if (!p || !dp) return VLLM_EINVAL;
  if (!vllm_aligned(p, 16) || !vllm_aligned(dp, 16)) return VLLM_EALIGN;
  const long long rows = n_mat * T;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  return with_vpt<256, 1, 2, 4>(T / 8, [&](auto vpt, auto) {
    attn_ds_kernel<decltype(vpt)::value><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)p,
                                                                                         (__nv_bfloat16*)dp, ld, T, scale);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

int vllm_ce_loss_f32(const float* logits, long long ld, const int64_t* labels, const int64_t* n_valid, long long rows, int vocab,
                     float* loss_sum, void* dlogits, long long ldd, void* stream) {
  if (rows < 0 || vocab <= 0 || ld < vocab) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!logits || !labels || !loss_sum || (dlogits && (!n_valid || ldd < vocab))) return VLLM_EINVAL;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  ce_loss_kernel<<<(unsigned)rows, 512, 0, (cudaStream_t)stream>>>(logits, ld, labels, n_valid, vocab, loss_sum,
                                                                   (__nv_bfloat16*)dlogits, ldd);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_scale_rows_bf16(void* x, long long ld, long long rows, int cols, const float* scale, void* stream) {
  if (rows < 0 || cols < 0 || ld < cols) return VLLM_EINVAL;
  if (rows == 0 || cols == 0) return VLLM_OK;
  if (!x || !scale) return VLLM_EINVAL;
  if (ld % 8 || !vllm_aligned(x, 16)) return VLLM_EALIGN;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  scale_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)x, ld, cols, scale);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_softmax_causal_len_bf16(void* s, long long ld, long long n_mat, int heads_per_batch, int T, const int* lens,
                                 float scale, void* stream) {
  if (n_mat < 0 || T <= 0 || T % 8 || ld < T || ld % 8 || heads_per_batch <= 0 || n_mat % heads_per_batch) return VLLM_EINVAL;
  if (n_mat == 0) return VLLM_OK;
  if (!s || !lens) return VLLM_EINVAL;
  if (!vllm_aligned(s, 16)) return VLLM_EALIGN;
  const long long rows = n_mat * T;
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  return with_vpt<256, 1, 2, 4>(T / 8, [&](auto vpt, auto) {
    softmax_causal_kernel<decltype(vpt)::value><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)s, ld, T, scale,
                                                                                                lens, heads_per_batch);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

int vllm_head_stack_qkv_pad_bf16(void* packed, long long ld, void* q, void* k, void* v, int batch, int tokens, int tokens_pad,
                                 int nq, int nkv, int head_dim, int to_stacked, void* stream) {
  if (batch < 0 || tokens < 0 || tokens_pad < tokens || nq <= 0 || nkv < 0 || head_dim <= 0 || (nkv && nq % nkv))
    return VLLM_EINVAL;
  if (ld < (long long)(nq + 2 * nkv) * head_dim) return VLLM_EINVAL;
  if ((long long)batch * tokens_pad == 0) return VLLM_OK;
  if (!packed || !q || (nkv && (!k || !v))) return VLLM_EINVAL;
  if (head_dim % 8) return VLLM_EUNSUPPORTED;                 // before n_vec: head_dim < 8 would give no vectors at all
  const long long n_vec = (long long)batch * tokens_pad * (nq + 2 * nkv) * (head_dim / 8);
  if (ld % 8 || !vllm_aligned(packed, 16) || !vllm_aligned(q, 16) || !vllm_aligned(k, 16) || !vllm_aligned(v, 16))
    return VLLM_EALIGN;
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  head_stack_qkv_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((uint4*)packed, ld / 8, (uint4*)q, (uint4*)k,
                                                                           (uint4*)v, batch, tokens, tokens_pad, nq, nkv,
                                                                           head_dim / 8, to_stacked ? 1 : 0, n_vec);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

static int gelu_launch(bool backward, const void* u, long long ldu, const void* dy, long long lddy, void* out, long long ldo,
                       long long rows, int cols, void* stream) {
  if (rows < 0 || cols <= 0 || cols % 8) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!u || !out || (backward && !dy)) return VLLM_EINVAL;
  if (ldu % 8 || ldo % 8 || (backward && lddy % 8) || !vllm_aligned(u, 16) || !vllm_aligned(out, 16) ||
      (backward && !vllm_aligned(dy, 16)))
    return VLLM_EALIGN;
  long long blocks = (rows * (cols / 8) + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (backward)
    gelu_kernel<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)u, ldu, (const __nv_bfloat16*)dy,
                                                                          lddy, (__nv_bfloat16*)out, ldo, rows, cols);
  else
    gelu_kernel<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)u, ldu, nullptr, 0,
                                                                           (__nv_bfloat16*)out, ldo, rows, cols);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_gelu_fwd_bf16(const void* u, long long ldu, void* y, long long ldy, long long rows, int cols, void* stream) {
  return gelu_launch(false, u, ldu, nullptr, 0, y, ldy, rows, cols, stream);
}

int vllm_gelu_bwd_bf16(const void* u, long long ldu, const void* dy, long long lddy, void* dx, long long lddx, long long rows,
                       int cols, void* stream) {
  return gelu_launch(true, u, ldu, dy, lddy, dx, lddx, rows, cols, stream);
}

int vllm_bias_grad_bf16(const void* dy, long long ldy, float* dbias, float* partials, int n_partials, long long rows, int cols,
                        void* stream) {
  if (rows < 0 || cols <= 0 || cols % 8) return VLLM_EINVAL;
  if (!dbias) return VLLM_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    return (int)cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)cols, st);
  }
  if (!dy || !partials) return VLLM_EINVAL;
  if (ldy % 8 || !vllm_aligned(dy, 16) || !vllm_aligned(partials, 16)) return VLLM_EALIGN;
  const int rows_per_cta = (int)((rows + (long long)vllm_num_sms() * 8 - 1) / ((long long)vllm_num_sms() * 8));
  const int blocks = rmsnorm_bwd_ctas(rows);
  if (n_partials < blocks) return VLLM_EINVAL;
  colsum_rows_kernel<<<dim3((unsigned)blocks, (unsigned)((cols / 8 + 255) / 256)), 256, 0, st>>>(
      (const __nv_bfloat16*)dy, ldy, rows, cols, rows_per_cta, partials);
  VLLM_CHECK_LAUNCH();
  colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials, dbias, blocks, cols);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_layernorm_bwd_wb_bf16(const void* x, long long ldx, const void* dy, long long ldy, float* dweight, float* dbias,
                               float* partials, int n_partials, long long rows, int cols, float eps, void* stream) {
  if (rows < 0 || cols <= 0 || cols % 8) return VLLM_EINVAL;
  if (!dweight || !dbias) return VLLM_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    const cudaError_t e = cudaMemsetAsync(dweight, 0, sizeof(float) * (size_t)cols, st);
    return (int)(e != cudaSuccess ? e : cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)cols, st));
  }
  if (!x || !dy || !partials) return VLLM_EINVAL;
  if (ldx % 8 || ldy % 8 || !vllm_aligned(x, 16) || !vllm_aligned(dy, 16) || !vllm_aligned(partials, 16)) return VLLM_EALIGN;
  const int rows_per_cta = (int)((rows + (long long)vllm_num_sms() * 8 - 1) / ((long long)vllm_num_sms() * 8));
  const int blocks = rmsnorm_bwd_ctas(rows);
  if (n_partials < blocks) return VLLM_EINVAL;
  return with_vpt<256, 1, 2, 4, 8>(cols / 8, [&](auto vpt, auto) {
    layernorm_bwd_wb_kernel<decltype(vpt)::value><<<(unsigned)blocks, 256, 0, st>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)dy, ldy, rows, cols, eps, rows_per_cta, partials);
    VLLM_CHECK_LAUNCH();
    colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials, dweight, blocks, cols);
    VLLM_CHECK_LAUNCH();
    colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials + (size_t)blocks * cols, dbias, blocks, cols);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

static int ln_gelu_bwd_rows_per_slot(long long rows) {
  const long long target = (long long)vllm_num_sms() * 32;
  return (int)((rows + target - 1) / target);
}

/* rows of dweight (and again of dbias) partials vllm_layernorm_gelu_bwd_bf16 needs for `rows` activation rows */
long long vllm_layernorm_gelu_bwd_partials(long long rows) {
  if (rows <= 0) return 0;
  const int rps = ln_gelu_bwd_rows_per_slot(rows);
  return (rows + rps - 1) / rps;
}

int vllm_layernorm_gelu_bwd_bf16(const void* x, long long ldx, const void* weight, const void* bias, const void* dy,
                                 long long ldy, void* dx, long long lddx, float* dweight, float* dbias, float* partials,
                                 long long n_partials, long long rows, int cols, float eps, void* stream) {
  if (rows < 0 || cols <= 0) return VLLM_EINVAL;
  if (cols % 8 || cols > 8 * 256 * 8) return VLLM_EUNSUPPORTED;
  if (!dweight || !dbias) return VLLM_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    const cudaError_t e = cudaMemsetAsync(dweight, 0, sizeof(float) * (size_t)cols, st);
    return (int)(e != cudaSuccess ? e : cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)cols, st));
  }
  if (!x || !weight || !bias || !dy || !dx || !partials) return VLLM_EINVAL;
  if (ldx % 8 || ldy % 8 || lddx % 8 || !vllm_aligned(x, 16) || !vllm_aligned(weight, 16) || !vllm_aligned(bias, 16) ||
      !vllm_aligned(dy, 16) || !vllm_aligned(dx, 16) || !vllm_aligned(partials, 16))
    return VLLM_EALIGN;
  const int rps = ln_gelu_bwd_rows_per_slot(rows);
  const long long slots = vllm_layernorm_gelu_bwd_partials(rows);
  if (n_partials < slots) return VLLM_EINVAL;
  auto go = [&](auto vpt, auto tpr) -> int {
    constexpr int VPT = decltype(vpt)::value, TPR = decltype(tpr)::value;
    const long long blocks = (slots + 256 / TPR - 1) / (256 / TPR);
    layernorm_gelu_bwd_kernel<VPT, TPR><<<(unsigned)blocks, 256, 0, st>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)weight, (const __nv_bfloat16*)bias, (const __nv_bfloat16*)dy, ldy,
        (__nv_bfloat16*)dx, lddx, rows, cols, eps, rps, slots, partials);
    VLLM_CHECK_LAUNCH();
    colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials, dweight, (int)slots, cols);
    VLLM_CHECK_LAUNCH();
    colsum_partials_kernel<<<(unsigned)((cols + 31) / 32), 256, 0, st>>>(partials + (size_t)slots * cols, dbias, (int)slots, cols);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  };
  // the forward's ladder (fused_ops.cu launch_norm): the statistics' reduction order, hence their bits, follow TPR
  const int nvec = cols / 8;
  if (nvec <= 128) return with_vpt<32, 1, 2, 4>(nvec, go);
  if (nvec <= 1024) return with_vpt<128, 2, 4, 8>(nvec, go);
  return with_vpt<256, 8>(nvec, go);
}

int vllm_point_pool_bwd_bf16(const float* loc, const float* weight, const float* counts, int n_points, const void* grad,
                             int levels, int regions, int height, int width, int channels, float* density, void* d_map,
                             void* stream) {
  if (n_points < 0 || levels <= 0 || regions < 0 || height <= 0 || width <= 0 || channels <= 0) return VLLM_EINVAL;
  if (channels % 8) return VLLM_EUNSUPPORTED;
  if (regions == 0) return VLLM_OK;
  if (!counts || !grad || !density || !d_map || (n_points > 0 && (!loc || !weight))) return VLLM_EINVAL;
  if (!vllm_aligned(grad, 16) || !vllm_aligned(d_map, 16) || (n_points > 0 && !vllm_aligned(loc, 8))) return VLLM_EALIGN;
  const long long HW = (long long)height * width;
  if (HW > 2147483647LL || regions > 65535 || levels > 65535) return VLLM_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  point_density_kernel<<<dim3((unsigned)((HW + 255) / 256), (unsigned)regions, (unsigned)levels), 256, 0, st>>>(
      loc, weight, n_points, regions, height, width, density);
  VLLM_CHECK_LAUNCH();
  long long blocks = ((long long)regions * HW * (channels / 8) + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  point_pool_outer_kernel<<<(unsigned)blocks, 256, 0, st>>>(density, counts, (const __nv_bfloat16*)grad, levels, regions, HW,
                                                            channels, (__nv_bfloat16*)d_map);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_assemble_embeds_bwd_bf16(const int* dest, const int* order, long long n, const void* d_embeds, int hidden,
                                  void* d_sources, long long source_rows, void* stream) {
  if (n < 0 || source_rows < 0 || hidden <= 0 || hidden % 8) return VLLM_EINVAL;
  if (source_rows == 0) return VLLM_OK;
  if (!d_sources || (n > 0 && (!dest || !order || !d_embeds))) return VLLM_EINVAL;
  if (!vllm_aligned(d_sources, 16) || (n > 0 && !vllm_aligned(d_embeds, 16))) return VLLM_EALIGN;
  long long blocks = source_rows;
  const long long cap = (long long)vllm_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  segment_sum_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dest, order, n, (const __nv_bfloat16*)d_embeds,
                                                                              hidden, (__nv_bfloat16*)d_sources, source_rows);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // extern "C"
