// Depthwise KxK convolution over a channels-last map (bf16 in/out, fp32 accumulate), stride 1, "same" padding.
//
// Replaces the cuDNN call behind `nn.Conv2d(channels, channels, kernel_size=dw_kernel_size, padding=(k-1)//2,
// groups=channels)` at the head of the reference DCNv3 module (visionllmv2/model/ops_dcnv3/modules/dcnv3.py:252-259;
// InternImage-H uses dw_kernel_size = 5, grounding_dino/modeling_ov_grounding_dino_mask_dn.py:5154-5170).  The
// reference permutes NHWC -> NCHW for the conv and back for the LayerNorm that follows; here the map stays
// channels-last: a thread owns 8 consecutive channels (one 16-byte vector) of TW consecutive pixels of a row, keeps
// the K input rows' strip of TW + K - 1 vectors in registers and reuses it for every horizontal tap, so each input
// vector is loaded K times (once per vertical tap) instead of K*K times.  Consecutive threads take consecutive
// channel vectors: every load is a coalesced run of the pixel's C*2 bytes.
//
//   y[n,h,w,c] = bias[c] + sum_{dy,dx} wt[dy*K+dx][c] * x[n, h+dy-K/2, w+dx-K/2, c]      (zeros outside the map)
//
// wt is the Conv2d weight [C,1,K,K] repacked tap-major [K*K][C] by the host wrapper (ops.dwconv_nhwc).
#include "rows.cuh"

namespace {

template <int K, int TW>
__global__ void __launch_bounds__(128)
dwconv_nhwc_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ wt,
                   const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int N, int H, int W, int C,
                   long long total) {
  constexpr int R = K / 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int CV = C / 8, WT = (W + TW - 1) / TW;
  const int cv = (int)(idx % CV);
  long long t = idx / CV;
  const int wt_i = (int)(t % WT); t /= WT;
  const int h = (int)(t % H);
  const int n = (int)(t / H);
  const int w0 = wt_i * TW;
  float acc[TW][8];
  {
    float b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = 0.f;
    if (bias) unpack8(__ldg(reinterpret_cast<const uint4*>(bias) + cv), b);
#pragma unroll
    for (int p = 0; p < TW; ++p)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[p][j] = b[j];
  }
  const __nv_bfloat16* xn = x + (size_t)n * H * W * C + cv * 8;
#pragma unroll 1
  for (int dy = 0; dy < K; ++dy) {
    const int hy = h + dy - R;
    if (hy < 0 || hy >= H) continue;
    float in[TW + K - 1][8];
#pragma unroll
    for (int j = 0; j < TW + K - 1; ++j) {
      const int wx = w0 + j - R;
      if (wx >= 0 && wx < W) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(xn + ((size_t)hy * W + wx) * C)), in[j]);
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) in[j][c] = 0.f;
      }
    }
#pragma unroll
    for (int dx = 0; dx < K; ++dx) {
      float wv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(wt + (size_t)(dy * K + dx) * C) + cv), wv);
#pragma unroll
      for (int p = 0; p < TW; ++p)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[p][c] = fmaf(in[p + dx][c], wv[c], acc[p][c]);
    }
  }
  __nv_bfloat16* yr = y + (((size_t)n * H + h) * W) * C + cv * 8;
#pragma unroll
  for (int p = 0; p < TW; ++p)
    if (w0 + p < W) *reinterpret_cast<uint4*>(yr + (size_t)(w0 + p) * C) = pack8(acc[p]);
}

template <int K>
int launch_dw(const void* x, const void* wt, const void* bias, void* y, int N, int H, int W, int C, cudaStream_t st) {
  constexpr int TW = 4;
  const long long total = (long long)N * H * ((W + TW - 1) / TW) * (C / 8);
  const long long blocks = (total + 127) / 128;
  if (blocks > 2147483647LL) return VLLM_EUNSUPPORTED;
  dwconv_nhwc_kernel<K, TW><<<(unsigned)blocks, 128, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)wt,
                                                              (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, N, H, W, C,
                                                              total);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // namespace

extern "C" int vllm_dwconv_nhwc_bf16(const void* x, const void* weight_taps, const void* bias, void* y, int batch,
                                     int height, int width, int channels, int kernel, void* stream) {
  if (batch < 0 || height < 0 || width < 0 || channels <= 0) return VLLM_EINVAL;
  if ((long long)batch * height * width == 0) return VLLM_OK;
  if (!x || !weight_taps || !y) return VLLM_EINVAL;
  if (channels % 8) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(x, 16) || !vllm_aligned(weight_taps, 16) || !vllm_aligned(y, 16) || (bias && !vllm_aligned(bias, 16)))
    return VLLM_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  switch (kernel) {
    case 3: return launch_dw<3>(x, weight_taps, bias, y, batch, height, width, channels, st);
    case 5: return launch_dw<5>(x, weight_taps, bias, y, batch, height, width, channels, st);
    case 7: return launch_dw<7>(x, weight_taps, bias, y, batch, height, width, channels, st);
    default: return VLLM_EUNSUPPORTED;
  }
}
