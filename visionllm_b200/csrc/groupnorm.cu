// GroupNorm over channels-last activations x[n, hw, c] (bf16 in/out, fp32 statistics), optional fused ReLU.
//
// Replaces nn.GroupNorm(32, d_model) after the 1x1 / 3x3 input projections of the Grounding-DINO neck
// (grounding_dino/modeling_ov_grounding_dino_mask_dn.py:2085-2110, applied at :2393-2405) and the
// detectron2 Conv2d(norm=GN[, activation=relu]) blocks of the mask-feature FPN (:2126-2151, :2470-2478).
// The reference runs them NCHW through cuDNN/ATen; our projections are GEMMs over NHWC rows, so the norm
// reads and writes the same [pixels, channels] matrix the GEMM produced -- no layout change in between.
//
// HBM-bound: 1 read for the statistics + 1 read + 1 write for the apply pass (2 B each) = 6 B / element.
// Statistics are deterministic: per-chunk (sum, sum^2) partials in fp32, combined in double in a fixed order.
#include "rows.cuh"
#include "vllm_b200.h"

namespace {

constexpr int GN_THREADS = 256;
constexpr int GN_MAX_CHUNKS = 128;

// grid (chunks, n).  Thread t owns the channel octet (t % c8) of pixels t / c8, t / c8 + ppi, ...  Octets of one
// group are reduced through shared memory; partial[n][chunk][g] = (sum, sumsq).
// Source geometry (vllm_groupnorm_nhwc_bf16_grid): pixel p of image n is read at pixel index
// n * img_pitch + (p / w_valid) * w_pitch + p % w_valid -- the valid [H, W] corner of a padded [Hp, Wp] grid, as the
// implicit-GEMM 3x3 convolution leaves it.  w_valid == w_pitch is the plain contiguous case.
__device__ __forceinline__ long long gn_src(long long p, long long w_valid, long long w_pitch) {
  if (w_valid == w_pitch) return p;
  const long long r = p / w_valid;
  return r * w_pitch + (p - r * w_valid);
}

__global__ void __launch_bounds__(GN_THREADS) gn_stats_kernel(const __nv_bfloat16* __restrict__ x, float2* __restrict__ partial,
                                                              long long hw, int c, int groups, int chunks,
                                                              long long w_valid, long long w_pitch, long long img_pitch) {
  extern __shared__ float2 sh[];  // [pixels-per-iteration][c8]
  const int c8 = c >> 3, cpg8 = (c / groups) >> 3;
  const int ppi = GN_THREADS / c8;  // pixels per iteration
  const int oct = threadIdx.x % c8, prow = threadIdx.x / c8;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const long long per = (hw + chunks - 1) / chunks;
  const long long p0 = chunk * per, p1 = min(hw, p0 + per);
  float s = 0.f, ss = 0.f;
  if (prow < ppi) {
    const uint4* base = reinterpret_cast<const uint4*>(x + (long long)n * img_pitch * c) + oct;
    for (long long p = p0 + prow; p < p1; p += ppi) {
      float f[8];
      unpack8(__ldg(base + gn_src(p, w_valid, w_pitch) * c8), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s += f[i];
        ss = fmaf(f[i], f[i], ss);
      }
    }
    sh[prow * c8 + oct] = make_float2(s, ss);
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    double ds = 0.0, dss = 0.0;
    for (int r = 0; r < ppi; ++r)
      for (int o = 0; o < cpg8; ++o) {
        const float2 v = sh[r * c8 + threadIdx.x * cpg8 + o];
        ds += v.x;
        dss += v.y;
      }
    partial[((long long)n * chunks + chunk) * groups + threadIdx.x] = make_float2((float)ds, (float)dss);
  }
}

// grid (blocks, n).  Every CTA first folds the chunk partials of its image into (mean, rstd) per group.
__global__ void __launch_bounds__(GN_THREADS) gn_apply_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                              const __nv_bfloat16* __restrict__ gamma,
                                                              const __nv_bfloat16* __restrict__ beta,
                                                              const float2* __restrict__ partial, long long hw, int c, int groups,
                                                              int chunks, float eps, int relu, long long w_valid, long long w_pitch,
                                                              long long img_pitch) {
  __shared__ float2 stat[256];
  const int n = blockIdx.y;
  const int c8 = c >> 3, cpg = c / groups;
  for (int g = threadIdx.x; g < groups; g += GN_THREADS) {
    double ds = 0.0, dss = 0.0;
    for (int k = 0; k < chunks; ++k) {
      const float2 v = partial[((long long)n * chunks + k) * groups + g];
      ds += v.x;
      dss += v.y;
    }
    const double cnt = (double)hw * cpg, mean = ds / cnt;
    double var = dss / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    stat[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
  __syncthreads();
  const int oct = threadIdx.x % c8, prow = threadIdx.x / c8, ppi = GN_THREADS / c8;
  if (prow >= ppi) return;
  float ga[8], be[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + oct), ga);
  unpack8(__ldg(reinterpret_cast<const uint4*>(beta) + oct), be);
  const float2 st = stat[(oct * 8) / cpg];
  const uint4* xin = reinterpret_cast<const uint4*>(x + (long long)n * img_pitch * c) + oct;
  uint4* yout = reinterpret_cast<uint4*>(y + (long long)n * hw * c) + oct;
  // four pixels per thread and iteration: four independent 16-byte loads in flight (one load per iteration leaves the apply
  // pass latency-bound)
  const long long step = (long long)gridDim.x * ppi;
  for (long long p0 = (long long)blockIdx.x * ppi + prow; p0 < hw; p0 += 4 * step) {
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long p = p0 + u * step;
      if (p < hw) raw[u] = __ldg(xin + gn_src(p, w_valid, w_pitch) * c8);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long p = p0 + u * step;
      if (p >= hw) break;
      float f[8];
      unpack8(raw[u], f);
      uint4 o;
      __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // ATen's GroupNorm: y = (x - mean) * rstd * gamma + beta evaluated in fp32, rounded once.
        float a = (f[2 * i] - st.x) * st.y * ga[2 * i] + be[2 * i];
        float b = (f[2 * i + 1] - st.x) * st.y * ga[2 * i + 1] + be[2 * i + 1];
        if (relu) {
          a = fmaxf(a, 0.f);
          b = fmaxf(b, 0.f);
        }
        op[i] = __floats2bfloat162_rn(a, b);
      }
      yout[p * c8] = o;
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// FPN top-down step of the mask-feature head (modeling_ov_grounding_dino_mask_dn.py:2486-2492):
//   y = lateral + F.interpolate(top, size=lateral.shape[-2:], mode="bilinear", align_corners=False)
// over channels-last bf16 maps in ONE pass: ATen's upsample_bilinear2d arithmetic restated (scale = in / out,
// src = scale * (dst + 0.5) - 0.5 clamped at 0, 2 x 2 taps combined row-then-column in fp32, the result rounded to bf16
// like the bf16 upsample output) and the bf16 add.  torch runs this as upcast -> fp32 upsample -> permute / downcast -> add
// (~2 GB of traffic for a 256 x 256 x 256 x 8 map); this kernel reads `top` (L2-resident: 4 output pixels share every
// source pixel) and `lateral` once and writes the sum once.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
upsample_add_nhwc_kernel(const __nv_bfloat16* __restrict__ top, const __nv_bfloat16* __restrict__ lat,
                         __nv_bfloat16* __restrict__ out, int Hi, int Wi, int Ho, int Wo, int C, long long n_vec,
                         float scale_h, float scale_w, long long top_pitch, int pad) {
  const int cv = C / 8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long p = i / cv;
    const int x = (int)(p % Wo); p /= Wo;
    const int y = (int)(p % Ho);
    const long long b = p / Ho;
    const float sy = fmaxf(scale_h * ((float)y + 0.5f) - 0.5f, 0.f), sx = fmaxf(scale_w * ((float)x + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < Hi - 1 ? 1 : 0), x1 = x0 + (x0 < Wi - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const __nv_bfloat16* tb = top + (size_t)b * top_pitch + c8 * 8;
    const uint4 v00 = __ldg(reinterpret_cast<const uint4*>(tb + ((size_t)y0 * Wi + x0) * C));
    const uint4 v01 = __ldg(reinterpret_cast<const uint4*>(tb + ((size_t)y0 * Wi + x1) * C));
    const uint4 v10 = __ldg(reinterpret_cast<const uint4*>(tb + ((size_t)y1 * Wi + x0) * C));
    const uint4 v11 = __ldg(reinterpret_cast<const uint4*>(tb + ((size_t)y1 * Wi + x1) * C));
    const uint4 lv = *reinterpret_cast<const uint4*>(lat + (size_t)i * 8);
    const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(&v00);
    const __nv_bfloat162* bq = reinterpret_cast<const __nv_bfloat162*>(&v01);
    const __nv_bfloat162* cq = reinterpret_cast<const __nv_bfloat162*>(&v10);
    const __nv_bfloat162* d = reinterpret_cast<const __nv_bfloat162*>(&v11);
    const __nv_bfloat162* l2 = reinterpret_cast<const __nv_bfloat162*>(&lv);
    uint4 ov;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __bfloat1622float2(a[k]), fb = __bfloat1622float2(bq[k]), fc = __bfloat1622float2(cq[k]),
                   fd = __bfloat1622float2(d[k]), fl = __bfloat1622float2(l2[k]);
      const float ux = hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fd.x);
      const float uy = hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fd.y);
      const __nv_bfloat162 ub = __floats2bfloat162_rn(ux, uy);                 // the bf16 upsample output
      const float2 uf = __bfloat1622float2(ub);
      o2[k] = __floats2bfloat162_rn(fl.x + uf.x, fl.y + uf.y);               // lateral + up, one bf16 rounding
    }
    // pad > 0: the output is the interior of a zero-bordered [Ho + 2 pad, Wo + 2 pad] map (the next 3x3 convolution's input)
    const size_t o = pad ? ((((size_t)b * (Ho + 2 * pad) + y + pad) * (Wo + 2 * pad) + x + pad) * cv + c8) : (size_t)i;
    *reinterpret_cast<uint4*>(out + o * 8) = ov;
  }
}

extern "C" {

long long vllm_groupnorm_workspace_bytes(int batch, int groups) {
  return (long long)batch * GN_MAX_CHUNKS * groups * (long long)sizeof(float2);
}

int vllm_groupnorm_nhwc_bf16_grid(const void* x, void* y, const void* gamma, const void* beta, int batch, long long h, long long w,
                                  long long x_w_pitch, long long x_image_pitch, int channels, int groups, float eps, int relu,
                                  void* workspace, long long workspace_bytes, void* stream) {
  if (batch < 0 || h < 0 || w < 0 || channels <= 0 || groups <= 0) return VLLM_EINVAL;
  const long long hw = h * w;
  if (batch == 0 || hw == 0) return VLLM_OK;
  if (!x || !y || !gamma || !beta || !workspace) return VLLM_EINVAL;
  if (x_w_pitch < w || x_image_pitch < (h - 1) * x_w_pitch + w) return VLLM_EINVAL;
  if (channels % groups) return VLLM_EINVAL;
  const int cpg = channels / groups;
  // one thread per 8-channel vector; a vector must not straddle two groups; a pixel row must fit one CTA pass
  if (cpg % 8 || channels > 8 * GN_THREADS || groups > 256) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(x, 16) || !vllm_aligned(y, 16) || !vllm_aligned(gamma, 16) || !vllm_aligned(beta, 16)) return VLLM_EALIGN;
  const int c8 = channels / 8, ppi = GN_THREADS / c8;
  long long want = (hw + (long long)ppi * 8 - 1) / ((long long)ppi * 8);  // >= 8 iterations per chunk
  int chunks = (int)(want < 1 ? 1 : (want > GN_MAX_CHUNKS ? GN_MAX_CHUNKS : want));
  if (workspace_bytes < (long long)batch * chunks * groups * (long long)sizeof(float2)) return VLLM_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  gn_stats_kernel<<<dim3(chunks, batch), GN_THREADS, (size_t)ppi * c8 * sizeof(float2), st>>>(
      (const __nv_bfloat16*)x, (float2*)workspace, hw, channels, groups, chunks, w, x_w_pitch, x_image_pitch);
  VLLM_CHECK_LAUNCH();
  long long blocks = (hw + (long long)ppi * 4 - 1) / ((long long)ppi * 4);
  const long long cap = (long long)vllm_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  gn_apply_kernel<<<dim3((unsigned)blocks, batch), GN_THREADS, 0, st>>>(
      (const __nv_bfloat16*)x, (__nv_bfloat16*)y, (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta,
      (const float2*)workspace, hw, channels, groups, chunks, eps, relu, w, x_w_pitch, x_image_pitch);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_upsample_add_nhwc_bf16_ex(const void* top, long long top_image_pitch, const void* lateral, void* out, int batch, int in_h,
                                   int in_w, int out_h, int out_w, int channels, int out_pad, void* stream) {
  if (batch < 0 || in_h <= 0 || in_w <= 0 || out_h <= 0 || out_w <= 0 || channels <= 0 || out_pad < 0) return VLLM_EINVAL;
  if (top_image_pitch < (long long)in_h * in_w * channels) return VLLM_EINVAL;
  if (batch == 0) return VLLM_OK;
  if (!top || !lateral || !out) return VLLM_EINVAL;
  if (channels % 8) return VLLM_EUNSUPPORTED;
  if (top_image_pitch % 8 || !vllm_aligned(top, 16) || !vllm_aligned(lateral, 16) || !vllm_aligned(out, 16)) return VLLM_EALIGN;
  const long long n_vec = (long long)batch * out_h * out_w * (channels / 8);
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  upsample_add_nhwc_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)top, (const __nv_bfloat16*)lateral, (__nv_bfloat16*)out, in_h, in_w, out_h, out_w, channels, n_vec,
      (float)in_h / (float)out_h, (float)in_w / (float)out_w, top_image_pitch, out_pad);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // extern "C"
