// DCNv3 forward (InternImage's core operator) for sm_90a.
//
// Replaces `dcnv3_forward` of the reference extension module `DCNv3`
//   visionllmv2/model/ops_dcnv3/src/dcnv3.h:20-38 (pybind vision.cpp:14-17), host dcnv3_cuda.cu:21-85,
//   kernel src/cuda/dcnv3_im2col_cuda.cuh:32-80 (bilinear) and :216-277 (im2col loop)
// behind vllm_dcnv3_forward_f32 (include/vllm_b200.h).  Same gather pattern as MSDA with one level, kh*kw taps
// on a dilated grid, offsets in PIXEL units scaled by offset_scale, zero padding outside the (unpadded) input.
//
// Layout (identical to the reference): input [N, H_in, W_in, G*C] (NHWC), offset [N, H_out, W_out, G*K*2]
// (x, y per tap, taps ordered kernel_w-major: p = i*kernel_h + j), mask [N, H_out, W_out, G*K],
// out [N, H_out, W_out, G*C].
//
//  * dcnv3_fwd_strict_kernel: reference thread mapping (one thread per output scalar) and operation order with
//    every product/sum individually rounded -- bit-exact against oracle/dcnv3_oracle.c.
//  * dcnv3_fwd_warp_kernel (C == 32, K <= 32): the MSDA warp-gather design: one warp per (output pixel, group);
//    phase 1 one lane per tap does the location arithmetic once and leaves per-corner {byte offset, weight} in
//    a warp-private smem slab; phase 2 lane = (corner, channel quad), one LDG.128 per lane per tap, float4 FMA,
//    two shuffle rounds.  Output pixels are walked in 8x16 patches so neighbouring taps hit in L1.
#include "common.cuh"

namespace {

struct DcnGeom { int h_low, w_low; float lh, lw; int mask; };

// location arithmetic of dcnv3_im2col_cuda.cuh:236-262, un-contracted
struct DcnParams {
  int kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w;
  int group, gc, H_in, W_in, H_out, W_out;
  float offset_scale;
};

__device__ __forceinline__ DcnGeom dcn_geom(const DcnParams& p, int ow, int oh, int i, int j, float off_w, float off_h) {
  const int p0_w = ((p.dil_w * (p.kernel_w - 1)) >> 1) - p.pad_w + ow * p.stride_w;
  const int p0_h = ((p.dil_h * (p.kernel_h - 1)) >> 1) - p.pad_h + oh * p.stride_h;
  const float p0_w_ = __fsub_rn((float)p0_w, __fmul_rn((float)((p.dil_w * (p.kernel_w - 1)) >> 1), p.offset_scale));
  const float p0_h_ = __fsub_rn((float)p0_h, __fmul_rn((float)((p.dil_h * (p.kernel_h - 1)) >> 1), p.offset_scale));
  const float loc_w = __fadd_rn(p0_w_, __fmul_rn(__fadd_rn((float)(i * p.dil_w), off_w), p.offset_scale));
  const float loc_h = __fadd_rn(p0_h_, __fmul_rn(__fadd_rn((float)(j * p.dil_h), off_h), p.offset_scale));
  DcnGeom g; g.mask = 0; g.h_low = 0; g.w_low = 0; g.lh = 0.f; g.lw = 0.f;
  if (loc_h > -1.f && loc_w > -1.f && loc_h < (float)p.H_in && loc_w < (float)p.W_in) {
    const int h_low = (int)floorf(loc_h), w_low = (int)floorf(loc_w);
    g.h_low = h_low; g.w_low = w_low;
    g.lh = __fsub_rn(loc_h, (float)h_low); g.lw = __fsub_rn(loc_w, (float)w_low);
    int m = 1;
    if (h_low >= 0 && w_low >= 0) m |= 2;
    if (h_low >= 0 && w_low + 1 <= p.W_in - 1) m |= 4;
    if (h_low + 1 <= p.H_in - 1 && w_low >= 0) m |= 8;
    if (h_low + 1 <= p.H_in - 1 && w_low + 1 <= p.W_in - 1) m |= 16;
    g.mask = m;
  }
  return g;
}

__global__ void __launch_bounds__(256)
dcnv3_fwd_strict_kernel(long long n, const float* __restrict__ in, const float* __restrict__ off,
                        const float* __restrict__ msk, float* __restrict__ out, const DcnParams p) {
  const int K = p.kernel_h * p.kernel_w;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x; index < n; index += stride) {
    long long t = index;
    const int c = (int)(t % p.gc); t /= p.gc;
    const long long sampling_index = t;
    const int g = (int)(t % p.group); t /= p.group;
    const int ow = (int)(t % p.W_out); t /= p.W_out;
    const int oh = (int)(t % p.H_out); t /= p.H_out;
    const long long b = t;
    const int qs = p.group * p.gc;
    const float* im = in + b * (long long)p.H_in * p.W_in * qs + g * p.gc + c;
    long long wp = sampling_index * K;
    float col = 0.f;
    for (int i = 0; i < p.kernel_w; ++i)
      for (int j = 0; j < p.kernel_h; ++j, ++wp) {
        const DcnGeom ge = dcn_geom(p, ow, oh, i, j, off[2 * wp], off[2 * wp + 1]);
        if (ge.mask & 1) {
          const float hh = __fsub_rn(1.f, ge.lh), hw = __fsub_rn(1.f, ge.lw);
          const long long ws = qs, hs = (long long)p.W_in * qs;
          const long long o = ge.h_low * hs + ge.w_low * ws;
          const float v1 = (ge.mask & 2) ? im[o] : 0.f, v2 = (ge.mask & 4) ? im[o + ws] : 0.f;
          const float v3 = (ge.mask & 8) ? im[o + hs] : 0.f, v4 = (ge.mask & 16) ? im[o + hs + ws] : 0.f;
          float val = __fmul_rn(__fmul_rn(hh, hw), v1);
          val = __fadd_rn(val, __fmul_rn(__fmul_rn(hh, ge.lw), v2));
          val = __fadd_rn(val, __fmul_rn(__fmul_rn(ge.lh, hw), v3));
          val = __fadd_rn(val, __fmul_rn(__fmul_rn(ge.lh, ge.lw), v4));
          col = __fadd_rn(col, __fmul_rn(val, msk[wp]));
        }
      }
    out[index] = col;
  }
}

constexpr int TH = 8, TW = 16, NW = 16, QPW = TH * TW / NW;   // 8 output pixels per warp
constexpr int META_ROW = 32 + 2;

__global__ void __launch_bounds__(NW * 32)
dcnv3_fwd_warp_kernel(const float* __restrict__ in, const float* __restrict__ off, const float* __restrict__ msk,
                      float* __restrict__ out, const DcnParams p, int tiles_w) {
  constexpr int C = 32;
  __shared__ __align__(16) int2 s_meta[NW][4][META_ROW];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x % p.group, tile = blockIdx.x / p.group, b = blockIdx.y;
  const int ty = tile / tiles_w, tx = tile % tiles_w;
  const int K = p.kernel_h * p.kernel_w;
  const int G = (32 / K) < QPW ? (32 / K) : QPW;
  const int qs = p.group * C;
  const int corner = lane >> 3, cq = lane & 7;
  const char* vbl = reinterpret_cast<const char*>(in + (size_t)b * p.H_in * p.W_in * qs + g * C + cq * 4);
  const int g1 = lane / K, s1 = lane - g1 * K;
  const int i1 = s1 / p.kernel_h, j1 = s1 - i1 * p.kernel_h;      // taps are kernel_w-major

  auto pixel_of = [&](int t, int& oh, int& ow) -> bool {
    oh = ty * TH + t / TW; ow = tx * TW + t % TW;
    return oh < p.H_out && ow < p.W_out;
  };

  for (int t0 = 0; t0 < QPW; t0 += G) {
    int oh = 0, ow = 0;
    bool live = false;
    if (g1 < G && t0 + g1 < QPW) live = pixel_of(warp * QPW + t0 + g1, oh, ow);
    bool clean = true;
    {
      int2 meta[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) meta[c] = make_int2(-1, 0);
      if (live) {
        const size_t pix = ((size_t)b * p.H_out + oh) * p.W_out + ow;
        const size_t si = (pix * p.group + g) * K + s1;
        const float ox = __ldg(off + 2 * si), oy = __ldg(off + 2 * si + 1), wv = __ldg(msk + si);
        const DcnGeom ge = dcn_geom(p, ow, oh, i1, j1, ox, oy);
        clean = (ge.mask == 31);
        if (ge.mask & 1) {
          const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
          const int base = (ge.h_low * p.W_in + ge.w_low) * qs * 4;
          if (ge.mask & 2) meta[0] = make_int2(base, __float_as_int(hh * hw * wv));
          if (ge.mask & 4) meta[1] = make_int2(base + qs * 4, __float_as_int(hh * ge.lw * wv));
          if (ge.mask & 8) meta[2] = make_int2(base + p.W_in * qs * 4, __float_as_int(ge.lh * hw * wv));
          if (ge.mask & 16) meta[3] = make_int2(base + (p.W_in + 1) * qs * 4, __float_as_int(ge.lh * ge.lw * wv));
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) s_meta[warp][c][lane] = meta[c];
    }
    const unsigned dirty = __ballot_sync(0xffffffffu, !clean);
    const unsigned alive = __ballot_sync(0xffffffffu, live);
    __syncwarp();
    for (int gi = 0; gi < G && t0 + gi < QPW; ++gi) {
      if (!((alive >> (gi * K)) & 1u)) continue;
      int poh, pow_;
      pixel_of(warp * QPW + t0 + gi, poh, pow_);
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      const int2* mp = &s_meta[warp][corner][gi * K];
      const unsigned gmask = (K >= 32 ? 0xffffffffu : ((1u << K) - 1u)) << (gi * K);
      if ((dirty & gmask) == 0) {
#pragma unroll 3
        for (int s = 0; s < K; ++s) {
          const int2 me = mp[s];
          const float4 v = __ldg(reinterpret_cast<const float4*>(vbl + (unsigned)me.x));
          const float w = __int_as_float(me.y);
          acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
        }
      } else {
        for (int s = 0; s < K; ++s) {
          const int2 me = mp[s];
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (me.x >= 0) v = __ldg(reinterpret_cast<const float4*>(vbl + (unsigned)me.x));
          const float w = __int_as_float(me.y);
          acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
        }
      }
#pragma unroll
      for (int o = 8; o <= 16; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
      }
      if (corner == 0) {
        float* op = out + ((((size_t)b * p.H_out + poh) * p.W_out + pow_) * p.group + g) * C + cq * 4;
        __stcs(reinterpret_cast<float4*>(op), acc);
      }
    }
    __syncwarp();
  }
}

// Backward (dcnv3_col2im_bilinear + col2im kernels, dcnv3_im2col_cuda.cuh:82-147, 278-370): one warp per
// (output pixel, group); the location arithmetic of a tap is done once per warp (the reference repeats it in every
// channel thread), lanes own channels c, c+32, ...; grad_input through fp32 atomicAdd exactly like the reference,
// grad_offset / grad_mask reduced over the channels with warp shuffles (the reference serialises that sum through
// shared memory in thread 0).
__global__ void __launch_bounds__(256)
dcnv3_bwd_warp_kernel(long long n_pg, const float* __restrict__ in, const float* __restrict__ off,
                      const float* __restrict__ msk, const float* __restrict__ gout, float* __restrict__ gin,
                      float* __restrict__ goff, float* __restrict__ gmsk, const DcnParams p) {
  const int lane = threadIdx.x & 31;
  const int qs = p.group * p.gc;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long pg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pg < n_pg; pg += warps) {
    long long t = pg;
    const int g = (int)(t % p.group); t /= p.group;
    const int ow = (int)(t % p.W_out); t /= p.W_out;
    const int oh = (int)(t % p.H_out); t /= p.H_out;
    const long long ib = t * (long long)p.H_in * p.W_in * qs + g * p.gc;
    const float* go = gout + pg * p.gc;
    long long wp = pg * p.kernel_h * p.kernel_w;
    for (int i = 0; i < p.kernel_w; ++i)
      for (int j = 0; j < p.kernel_h; ++j, ++wp) {
        const DcnGeom ge = dcn_geom(p, ow, oh, i, j, off[2 * wp], off[2 * wp + 1]);
        float ga = 0.f, gw = 0.f, gh = 0.f;
        if (ge.mask & 1) {
          const float weight = msk[wp];
          const float hh = 1.f - ge.lh, hw = 1.f - ge.lw;
          const float w1 = hh * hw, w2 = hh * ge.lw, w3 = ge.lh * hw, w4 = ge.lh * ge.lw;
          const long long ws = qs, hs = (long long)p.W_in * qs, o1 = ib + ge.h_low * hs + ge.w_low * ws;
          for (int c = lane; c < p.gc; c += 32) {
            const float tg = go[c], tgi = tg * weight;
            float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f, dh = 0.f, dw = 0.f;
            if (ge.mask & 2) { v1 = in[o1 + c]; dh -= hw * v1; dw -= hh * v1; atomicAdd(gin + o1 + c, w1 * tgi); }
            if (ge.mask & 4) { v2 = in[o1 + ws + c]; dh -= ge.lw * v2; dw += hh * v2; atomicAdd(gin + o1 + ws + c, w2 * tgi); }
            if (ge.mask & 8) { v3 = in[o1 + hs + c]; dh += hw * v3; dw -= ge.lh * v3; atomicAdd(gin + o1 + hs + c, w3 * tgi); }
            if (ge.mask & 16) { v4 = in[o1 + hs + ws + c]; dh += ge.lw * v4; dw += ge.lh * v4; atomicAdd(gin + o1 + hs + ws + c, w4 * tgi); }
            ga += tg * (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
            gw += p.offset_scale * dw * tgi;
            gh += p.offset_scale * dh * tgi;
          }
        }
        ga = warp_sum(ga); gw = warp_sum(gw); gh = warp_sum(gh);
        if (lane == 0) { gmsk[wp] = ga; goff[2 * wp] = gw; goff[2 * wp + 1] = gh; }
      }
  }
}

}  // namespace

extern "C" int vllm_dcnv3_forward_f32(const float* input, const float* offset, const float* mask, float* out, int N,
                                      int H_in, int W_in, int H_out, int W_out, int group, int group_channels,
                                      int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                                      int dilation_h, int dilation_w, float offset_scale, int flags, void* stream) {
  if (N < 0 || H_in <= 0 || W_in <= 0 || H_out < 0 || W_out < 0 || group <= 0 || group_channels <= 0 ||
      kernel_h <= 0 || kernel_w <= 0 || stride_h <= 0 || stride_w <= 0 || dilation_h <= 0 || dilation_w <= 0)
    return VLLM_EINVAL;
  const long long n = (long long)N * H_out * W_out * group * group_channels;
  if (n == 0) return VLLM_OK;
  if (!input || !offset || !mask || !out) return VLLM_EINVAL;
  if ((long long)H_in * W_in * group * group_channels * 4 > 2147483647LL) return VLLM_EUNSUPPORTED;
  DcnParams p{kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
              group, group_channels, H_in, W_in, H_out, W_out, offset_scale};
  cudaStream_t st = (cudaStream_t)stream;
  const int K = kernel_h * kernel_w;
  if (!(flags & 1) && group_channels == 32 && K <= 32 && N <= 65535 && vllm_aligned(input, 16) && vllm_aligned(out, 16)) {
    const int tiles_w = (W_out + TW - 1) / TW, tiles_h = (H_out + TH - 1) / TH;
    dim3 grid((unsigned)(tiles_w * tiles_h * group), (unsigned)N);
    dcnv3_fwd_warp_kernel<<<grid, NW * 32, 0, st>>>(input, offset, mask, out, p, tiles_w);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  }
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)vllm_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  dcnv3_fwd_strict_kernel<<<(unsigned)blocks, 256, 0, st>>>(n, input, offset, mask, out, p);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

extern "C" int vllm_dcnv3_backward_f32(const float* input, const float* offset, const float* mask,
                                       const float* grad_output, float* grad_input, float* grad_offset,
                                       float* grad_mask, int N, int H_in, int W_in, int H_out, int W_out, int group,
                                       int group_channels, int kernel_h, int kernel_w, int stride_h, int stride_w,
                                       int pad_h, int pad_w, int dilation_h, int dilation_w, float offset_scale,
                                       void* stream) {
  if (N < 0 || H_in <= 0 || W_in <= 0 || H_out < 0 || W_out < 0 || group <= 0 || group_channels <= 0 ||
      kernel_h <= 0 || kernel_w <= 0 || stride_h <= 0 || stride_w <= 0 || dilation_h <= 0 || dilation_w <= 0)
    return VLLM_EINVAL;
  const long long n_pg = (long long)N * H_out * W_out * group;
  if (n_pg == 0) return VLLM_OK;
  if (!input || !offset || !mask || !grad_output || !grad_input || !grad_offset || !grad_mask) return VLLM_EINVAL;
  DcnParams p{kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
              group, group_channels, H_in, W_in, H_out, W_out, offset_scale};
  long long blocks = (n_pg + 7) / 8;
  const long long cap = (long long)vllm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  dcnv3_bwd_warp_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_pg, input, offset, mask, grad_output,
                                                                            grad_input, grad_offset, grad_mask, p);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}
