/* ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * CPU restatement of the reference DCNv3 forward as its CUDA kernel defines it:
 *   VisionLLMv2/visionllmv2/model/ops_dcnv3/src/cuda/dcnv3_im2col_cuda.cuh
 *     :32-80   bilinear corner gather; :216-277 im2col loop (taps kernel_w-major, pixel-unit offsets * offset_scale,
 *     range test, col += val * mask).
 * fp32, every product/sum individually rounded (-ffp-contract=off): the reference GPU build may contract some of
 * these into FMAs, so tap positions that land within 1 ulp of a cell edge can differ from IT; values are compared
 * with a tolerance, and the strict CUDA kernel matches THIS file bit for bit.
 * Pinned by tests/golden/dcnv3_ref_*.npz (outputs of the reference's own dcnv3_core_pytorch,
 * ops_dcnv3/functions/dcnv3_func.py:120-161, on the vectors of ops_dcnv3/test.py:20-60). */
#include <math.h>
#include <stdint.h>

void oracle_dcnv3_forward_f32(const float* in, const float* off, const float* msk, float* out, int N, int H_in,
                              int W_in, int H_out, int W_out, int group, int gc, int kh, int kw, int sh, int sw,
                              int ph, int pw, int dh, int dw, float offset_scale) {
  const int K = kh * kw, qs = group * gc;
  const long long pixels = (long long)N * H_out * W_out * group;
#pragma omp parallel for schedule(static)
  for (long long pg = 0; pg < pixels; ++pg) {
    long long t = pg;
    const int g = (int)(t % group); t /= group;
    const int ow = (int)(t % W_out); t /= W_out;
    const int oh = (int)(t % H_out); t /= H_out;
    const long long b = t;
    const int p0_w = ((dw * (kw - 1)) >> 1) - pw + ow * sw;
    const int p0_h = ((dh * (kh - 1)) >> 1) - ph + oh * sh;
    volatile float tw = (float)((dw * (kw - 1)) >> 1) * offset_scale, th = (float)((dh * (kh - 1)) >> 1) * offset_scale;
    const float p0_w_ = (float)p0_w - tw, p0_h_ = (float)p0_h - th;
    for (int c = 0; c < gc; ++c) {
      const float* im = in + b * (long long)H_in * W_in * qs + g * gc + c;
      long long wp = pg * K;
      float col = 0.f;
      for (int i = 0; i < kw; ++i)
        for (int j = 0; j < kh; ++j, ++wp) {
          volatile float aw = (float)(i * dw) + off[2 * wp], ah = (float)(j * dh) + off[2 * wp + 1];
          volatile float mw = aw * offset_scale, mh = ah * offset_scale;
          const float loc_w = p0_w_ + mw, loc_h = p0_h_ + mh;
          if (!(loc_h > -1 && loc_w > -1 && loc_h < H_in && loc_w < W_in)) continue;
          const int hl = (int)floorf(loc_h), wl = (int)floorf(loc_w);
          const float lh = loc_h - hl, lw = loc_w - wl, hh = 1 - lh, hw = 1 - lw;
          const long long ws = qs, hs = (long long)W_in * qs, o = hl * hs + wl * ws;
          const float v1 = (hl >= 0 && wl >= 0) ? im[o] : 0.f;
          const float v2 = (hl >= 0 && wl + 1 <= W_in - 1) ? im[o + ws] : 0.f;
          const float v3 = (hl + 1 <= H_in - 1 && wl >= 0) ? im[o + hs] : 0.f;
          const float v4 = (hl + 1 <= H_in - 1 && wl + 1 <= W_in - 1) ? im[o + hs + ws] : 0.f;
          const float val = (hh * hw) * v1 + (hh * lw) * v2 + (lh * hw) * v3 + (lh * lw) * v4;
          col += val * msk[wp];
        }
      out[pg * gc + c] = col;
    }
  }
}

/* Backward, restating dcnv3_col2im_bilinear and the col2im kernels (dcnv3_im2col_cuda.cuh:82-147, 278-370):
 * per (pixel, group, tap) the channel contributions to grad_offset / grad_mask are summed in channel order
 * (thread 0's loop, :349-356); grad_input accumulates (atomicAdd on the GPU, so its order is free there).
 * grad_input must be zeroed by the caller.  Pinned by tests/golden/dcnv3_bwd_*.npz (fp64 autograd through the
 * reference's own dcnv3_core_pytorch). */
#define DCN_BACKWARD(T, SUFFIX)                                                                                       \
  void oracle_dcnv3_backward_##SUFFIX(const T* in, const T* off, const T* msk, const T* gout, T* gin, T* goff,        \
                                      T* gmsk, int N, int H_in, int W_in, int H_out, int W_out, int group, int gc,    \
                                      int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, T offset_scale) { \
    const int K = kh * kw, qs = group * gc;                                                                           \
    const long long pixels = (long long)N * H_out * W_out * group;                                                    \
    for (long long pg = 0; pg < pixels; ++pg) {                                                                       \
      long long t = pg;                                                                                               \
      const int g = (int)(t % group); t /= group;                                                                     \
      const int ow = (int)(t % W_out); t /= W_out;                                                                    \
      const int oh = (int)(t % H_out); t /= H_out;                                                                    \
      const long long b = t, ib = b * (long long)H_in * W_in * qs + g * gc;                                           \
      const int p0_w = ((dw * (kw - 1)) >> 1) - pw + ow * sw;                                                         \
      const int p0_h = ((dh * (kh - 1)) >> 1) - ph + oh * sh;                                                         \
      volatile T tw = (T)((dw * (kw - 1)) >> 1) * offset_scale, th = (T)((dh * (kh - 1)) >> 1) * offset_scale;        \
      const T p0_w_ = (T)p0_w - tw, p0_h_ = (T)p0_h - th;                                                             \
      long long wp = pg * K;                                                                                          \
      for (int i = 0; i < kw; ++i)                                                                                    \
        for (int j = 0; j < kh; ++j, ++wp) {                                                                          \
          volatile T aw = (T)(i * dw) + off[2 * wp], ah = (T)(j * dh) + off[2 * wp + 1];                              \
          volatile T mw = aw * offset_scale, mh = ah * offset_scale;                                                  \
          const T loc_w = p0_w_ + mw, loc_h = p0_h_ + mh;                                                             \
          T ga = 0, gw = 0, gh = 0;                                                                                   \
          if (loc_h > -1 && loc_w > -1 && loc_h < H_in && loc_w < W_in) {                                             \
            const int hl = (int)floor((double)loc_h), wl = (int)floor((double)loc_w);                                 \
            const T lh = loc_h - hl, lw = loc_w - wl, hh = 1 - lh, hw = 1 - lw;                                       \
            const T w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;                                           \
            const long long ws = qs, hs = (long long)W_in * qs, o1 = ib + hl * hs + wl * ws;                          \
            const int m1 = hl >= 0 && wl >= 0, m2 = hl >= 0 && wl + 1 <= W_in - 1;                                    \
            const int m3 = hl + 1 <= H_in - 1 && wl >= 0, m4 = hl + 1 <= H_in - 1 && wl + 1 <= W_in - 1;              \
            for (int c = 0; c < gc; ++c) {                                                                            \
              const T tg = gout[pg * gc + c], tgi = tg * msk[wp];                                                     \
              T v1 = 0, v2 = 0, v3 = 0, v4 = 0, dhh = 0, dww = 0;                                                     \
              if (m1) { v1 = in[o1 + c]; dhh -= hw * v1; dww -= hh * v1; gin[o1 + c] += w1 * tgi; }                   \
              if (m2) { v2 = in[o1 + ws + c]; dhh -= lw * v2; dww += hh * v2; gin[o1 + ws + c] += w2 * tgi; }         \
              if (m3) { v3 = in[o1 + hs + c]; dhh += hw * v3; dww -= lh * v3; gin[o1 + hs + c] += w3 * tgi; }         \
              if (m4) { v4 = in[o1 + hs + ws + c]; dhh += lw * v4; dww += lh * v4; gin[o1 + hs + ws + c] += w4 * tgi; } \
              ga += tg * (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);                                                     \
              gw += offset_scale * dww * tgi;                                                                         \
              gh += offset_scale * dhh * tgi;                                                                         \
            }                                                                                                         \
          }                                                                                                           \
          gmsk[wp] = ga; goff[2 * wp] = gw; goff[2 * wp + 1] = gh;                                                    \
        }                                                                                                             \
    }                                                                                                                 \
  }

DCN_BACKWARD(float, f32)
DCN_BACKWARD(double, f64)
