/* libvllm_b200.so -- C-ABI of the H100-native (sm_90a) VisionLLMv2 forward hot path.
 *
 * Plain pointers and sizes only (no torch types).  All pointers are DEVICE
 * pointers unless the parameter name says `host`.  Every function is
 * re-entrant, keeps no global state (except the tuning knob marked below),
 * enqueues on the caller's `stream` (a cudaStream_t passed as void*) and never
 * allocates or synchronises.  Outputs are caller-allocated and fully written.
 *
 * Return value: 0 = ok; < 0 = argument error (VLLM_E*); > 0 = the cudaError_t
 * of a failed launch.  The reference only printf()s launch errors
 * (mmcv/ops/csrc/pytorch/cuda/ms_deform_attn_cuda.cu:41-44) and its Python
 * caller silently falls back to grid_sample (grounding_dino/
 * modeling_ov_grounding_dino_mask_dn.py:777-779); this boundary reports them.
 *
 * Paths below are relative to the VisionLLMv2/ directory of the reference project.
 */
#ifndef VLLM_B200_H
#define VLLM_B200_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define VLLM_OK 0
#define VLLM_EINVAL (-1)       /* null pointer / negative size / inconsistent shapes */
#define VLLM_EUNSUPPORTED (-2) /* shape outside what the kernels implement */
#define VLLM_EALIGN (-3)       /* pointer alignment the vector path needs is missing */

/* Library identity / build info: "vllm_b200 <git-less version> sm_90a". */
const char* vllm_version(void);

/* ---- Multi-scale deformable attention --------------------------------------
 * Replaces `ms_deform_attn_forward` of the reference extension module
 * `MultiScaleDeformableAttention`:
 *   visionllmv2/model/unipose/ops/src/ms_deform_attn.h:21-40 (pybind vision.cpp:13-16)
 *   mmcv/mmcv/ops/csrc/pytorch/ms_deform_attn.cpp:38-60 (pybind.cpp:788-798)
 *   kernel: mmcv/mmcv/ops/csrc/common/cuda/ms_deform_attn_cuda_kernel.cuh:17-64,200-254
 * value [batch, spatial_size, num_heads, channels]; spatial_shapes [num_levels,2]
 * int64 (H,W) on device; level_start_index [num_levels] int64 on device;
 * sampling_loc [batch, num_query, num_heads, num_levels, num_point, 2] (x,y);
 * attn_weight [batch, num_query, num_heads, num_levels, num_point];
 * out [batch, num_query, num_heads*channels].
 * host_shapes_hint: optional HOST copy of spatial_shapes (may be NULL); when given
 * it MUST equal spatial_shapes.  It orders the work (2-D pixel patches when
 * num_query == spatial_size) and sizes the window kernel's TMA maps; with a hint
 * equal to spatial_shapes the result is bit-identical to the NULL-hint result.
 * Any batch size: batches over 65535 images run as several launches.
 * flags bit0 (VLLM_MSDA_STRICT): reference thread mapping and summation order
 * with no FMA contraction -- bit-exact against oracle/msda_oracle.c.
 */
#define VLLM_MSDA_STRICT 1
int vllm_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                          const float* sampling_loc, const float* attn_weight, float* out, int batch,
                          int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                          int num_point, const int64_t* host_shapes_hint, int flags, void* stream);
/* "Fast mode" of the same operator (SURVEY 8d cfg 2b): value is bf16 [N,S,M,32] -- the bf16 value_proj output the
 * reference upcasts with .float() before calling its fp32-only kernel (modeling_ov_grounding_dino_mask_dn.py:764-766)
 * -- sampling_loc / attn_weight stay fp32, accumulation is fp32, out is fp32 or bf16 (out_bf16) [N,Lq,M*32].  Same
 * products as vllm_msda_forward_f32 on the upcast value (bf16 -> fp32 is exact), summed in another order: each lane
 * sums every second sample and a 4 + 2 + 1 shuffle tree joins them, so results are bit-identical to _f32 only for
 * levels*points == 1 and otherwise agree within the fp32 reassociation bound of both.  A bf16 out is the fp32 result
 * rounded to nearest.  channels == 32, levels*points <= 32, else VLLM_EUNSUPPORTED; value / out not 16-byte or
 * sampling_loc not 8-byte aligned: VLLM_EALIGN. */
int vllm_msda_forward_bf16v(const void* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                            const float* sampling_loc, const float* attn_weight, void* out, int out_bf16, int batch,
                            int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                            int num_point, const int64_t* host_shapes_hint, void* stream);
/* fp64 instance of the same operator (AT_DISPATCH_FLOATING_TYPES,
 * ms_deform_attn_cuda.cu:258); always the strict kernel. */
int vllm_msda_forward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                          const double* sampling_loc, const double* attn_weight, double* out, int batch,
                          int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                          int num_point, void* stream);
/* Backward of the same operator (`ms_deform_attn_backward`, unipose ops/src/ms_deform_attn.h:42-62; mmcv
 * pybind.cpp:793-798; kernels ms_deform_attn_cuda_kernel.cuh:66-124,256-801).  grad_output [batch, num_query,
 * num_heads*channels].  grad_value MUST be zero-initialised by the caller (corner contributions are accumulated
 * with atomics, like the reference); grad_sampling_loc / grad_attn_weight are fully written. */
int vllm_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                           const float* sampling_loc, const float* attn_weight, const float* grad_output,
                           float* grad_value, float* grad_sampling_loc, float* grad_attn_weight, int batch,
                           int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                           int num_point, void* stream);
int vllm_msda_backward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                           const double* sampling_loc, const double* attn_weight, const double* grad_output,
                           double* grad_value, double* grad_sampling_loc, double* grad_attn_weight, int batch,
                           int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                           int num_point, void* stream);
/* Parity instrumentation: for each of n_samples = batch*num_query*num_heads*
 * num_levels*num_point samples writes (h_low, w_low, mask) int32 triples using
 * the SAME device function the forward kernels use.  mask bit0 = sample in
 * range (kernel.cuh:241), bits1..4 = corner in bounds (kernel.cuh:39-57).
 * h_low/w_low are 0 when bit0 is clear. */
int vllm_msda_sample_indices_f32(const int64_t* spatial_shapes, const float* sampling_loc, int32_t* out_hwm,
                                 long long n_samples, int num_levels, int num_point, void* stream);
/* Path selection for tests and benchmarks (process-global, not part of the drop-in API).  Every value forces a path
 * the library also takes by itself on other inputs, so a test can compare two paths on one input:
 *   VLLM_MSDA_DEFAULT         the dispatch described here
 *   VLLM_MSDA_NO_HINT         vllm_msda_forward_f32 ignores host_shapes_hint (linear query tiles instead of 2-D pixel
 *                             patches: what a caller that passes NULL gets)
 *   VLLM_MSDA_BF16_NO_WINDOW  vllm_msda_forward_bf16v skips the window kernel and runs the warp-gather kernel, as it does
 *                             for shapes the window kernel does not cover
 *   VLLM_MSDA_FP32_WINDOW     vllm_msda_forward_f32 (non-strict) tries the window kernel first
 * Any other value: VLLM_EINVAL, nothing changes. */
#define VLLM_MSDA_DEFAULT 0
#define VLLM_MSDA_NO_HINT 4
#define VLLM_MSDA_BF16_NO_WINDOW 32
#define VLLM_MSDA_FP32_WINDOW 33
int vllm_msda_set_variant(int variant);
/* Encoder shape (num_query == spatial_size, host_shapes_hint given, <= 4 levels, channels == 32): vllm_msda_forward_bf16v
 * -- and vllm_msda_forward_f32 (non-strict) under VLLM_MSDA_FP32_WINDOW -- run the TMA-staged window kernel
 * (csrc/msda_win.cu): one CTA per (image region, head) loads the bounded value window of every level into shared memory
 * with cp.async.bulk.tensor (zero fill outside the map = the operator's zero padding) and gathers from there; a (query,
 * head) with a sample outside its window falls back to the global-memory path inside the same kernel (bit-identical
 * sums).  vllm_msda_set_window: tuning knob (process-global) -- level-0 patch height / width in pixels and level-0 halo;
 * 0 = default (16 x 32, halo 8 for bf16 rows; 8 x 8, halo 6 for fp32). */
int vllm_msda_set_window(int patch_h, int patch_w, int halo0);
/* Window fill of the encoder kernel: bit l of `tma` set = level l's window arrives as one TMA box (cp.async.bulk.tensor.5d),
 * clear = cooperative cp.async (one 64 / 128-byte row per thread and step); 1 = every level by TMA (its r2 meaning),
 * 0 = every level by cp.async, negative = the measured default.  Same results for every mix: the TMA form is request-rate
 * bound on 64-byte rows, the cooperative form costs issue slots of an issue-bound kernel (DESIGN 6.2). */
int vllm_msda_set_window_fill(int tma);
/* The deformable-attention MODULE's inner part in one kernel (GroundingDinoMultiscaleDeformableAttention.forward,
 * modeling_ov_grounding_dino_mask_dn.py:742-776, encoder shape, 4 levels x 4 points, channels 32): qp [batch, num_query,
 * ld_qp] bf16 = the packed sampling_offsets | attention_weights projection output (M*K*2 offsets then M*K logits per row),
 * reference_points [batch, num_query, num_levels, 2] fp32.  Does the softmax over the 16 logits, offset / (W, H) in bf16,
 * reference + offset in fp32 with torch's exact arithmetic, then the window gather of vllm_msda_forward_bf16v; optionally
 * writes the bf16 attention weights [batch, num_query, M, 16] the module returns.  VLLM_EUNSUPPORTED when the window
 * path does not apply (the caller keeps the unfused path). */
int vllm_msda_forward_fused_bf16(const void* value, const int64_t* level_start_index, const void* qp, int ld_qp,
                                 const float* reference_points, void* out, int out_bf16, void* attn_weights_out, int batch,
                                 int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                                 const int64_t* host_shapes_hint, void* stream);

/* ---- DCNv3 forward (InternImage core op) ------------------------------------------
 * Replaces `dcnv3_forward` of the reference extension module `DCNv3`
 * (visionllmv2/model/ops_dcnv3/src/dcnv3.h:20-38, vision.cpp:14-17; kernel
 * src/cuda/dcnv3_im2col_cuda.cuh:32-80,216-277; caller functions/dcnv3_func.py:39-58).
 * input [N,H_in,W_in,group*group_channels] (NHWC), offset [N,H_out,W_out,group*K*2] (x,y per
 * tap, taps kernel_w-major), mask [N,H_out,W_out,group*K], out [N,H_out,W_out,group*
 * group_channels]; K = kernel_h*kernel_w; offsets are in pixels and scaled by offset_scale.
 * flags bit0: strict kernel (reference thread mapping, no FMA contraction; bit-exact vs
 * oracle/dcnv3_oracle.c).  fp32 only (the reference module always upcasts,
 * ops_dcnv3/modules/dcnv3.py:331-340). */
int vllm_dcnv3_forward_f32(const float* input, const float* offset, const float* mask, float* out, int N,
                           int H_in, int W_in, int H_out, int W_out, int group, int group_channels,
                           int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                           int dilation_h, int dilation_w, float offset_scale, int flags, void* stream);

/* DCNv3 backward: `dcnv3_backward` of the same extension module (dcnv3.h:40-59; col2im kernels
 * dcnv3_im2col_cuda.cuh:82-147,278-370; caller functions/dcnv3_func.py:60-77).  grad_input [N,H_in,W_in,G*C] MUST
 * be zero-filled by the caller (accumulated with atomicAdd like the reference, dcnv3_cuda.cu:131 at::zeros_like);
 * grad_offset / grad_mask are written in full. */
int vllm_dcnv3_backward_f32(const float* input, const float* offset, const float* mask, const float* grad_output,
                            float* grad_input, float* grad_offset, float* grad_mask, int N, int H_in, int W_in,
                            int H_out, int W_out, int group, int group_channels, int kernel_h, int kernel_w,
                            int stride_h, int stride_w, int pad_h, int pad_w, int dilation_h, int dilation_w,
                            float offset_scale, void* stream);

/* ---- bf16 tensor-core GEMM with fused epilogue (wgmma / TMA / mbarrier) ----------
 * C[M, n_out] = epi(A[M,K] . B[N,K]^T): every nn.Linear on the hot path
 * (internvit/modeling_intern_vit.py:112,124,172-173; modeling_visionllmv2.py:162-184;
 * HF LlamaDecoderLayer / internlm2/modeling_internlm2.py:235-360;
 * grounding_dino/modeling_ov_grounding_dino_mask_dn.py:674-677,1116-1117), replacing
 * torch's cuBLAS calls plus the separate bias / activation / LayerScale / residual
 * elementwise kernels.  A, B bf16 row-major with row pitches lda, ldb (elements,
 * multiples of 8, 16-byte aligned bases).  epilogue order: +bias[N] (bf16, may be
 * NULL) -> act -> *colscale[N] (bf16, may be NULL) -> +residual[M, ldr] (bf16, may be
 * NULL) -> store bf16 (out_f32 = 0) or fp32 (out_f32 = 1) with row pitch ldc.
 * act: 0 none, 1 GELU(erf), 2 ReLU, 3 SiLU, 4 SwiGLU (columns (2j,2j+1) = (gate_j,
 * up_j) -> n_out = N/2 = silu(gate)*up), 5 quick-GELU (CLIP). */
#define VLLM_ACT_NONE 0
#define VLLM_ACT_GELU 1
#define VLLM_ACT_RELU 2
#define VLLM_ACT_SILU 3
#define VLLM_ACT_SWIGLU 4
#define VLLM_ACT_QUICKGELU 5
int vllm_gemm_bf16(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                   const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                   void* stream);
/* Same GEMM with a row mask: rows m with row_keep[m] == 0 are stored as exact zeros whatever the epilogue computed --
 * `value = value_proj(x).masked_fill(~attention_mask[..., None], 0)` of the deformable-attention module
 * (modeling_ov_grounding_dino_mask_dn.py:729-732) without the extra read + write of `value`.  Not with SwiGLU. */
int vllm_gemm_bf16_rowmask(const void* A, int lda, const void* B, int ldb, void* C, int ldc, int M, int N, int K,
                           const void* bias, const void* colscale, const void* residual, int ldr, int act, int out_f32,
                           const unsigned char* row_keep, void* stream);
/* SM budgets of the persistent GEMM grid (process-global; 0 = every SM): `all_gemms` caps every launch, `scatter_gemm` the
 * scatter GEMM alone.  A GEMM CTA owns its SM, so the link-bound exchange kernels of another stream (tensor-parallel
 * micro-batches, visionllm_b200/tp.py) overlap a GEMM only on SMs its grid leaves free. */
int vllm_gemm_set_sm_limit(int all_gemms, int scatter_gemm);
/* Stride-1 KxK convolution over a zero-padded channels-last map as ONE implicit GEMM (no im2col buffer): the 3x3
 * `output_convs` of the Grounding-DINO mask-feature FPN (modeling_ov_grounding_dino_mask_dn.py:2136-2146, :2476).
 * xpad: [pad_pixels, channels] bf16 = the padded images flattened (image rows of `padded_width` pixels, images back
 * to back); weight [out_channels, kernel_h*kernel_w*channels] in (dy, dx, c) order, pitch ldw.  Row i of `out`
 * ([pad_pixels, out_channels], pitch ldo) is the window whose TOP-LEFT tap is padded pixel i; the caller keeps the rows
 * whose window lies inside one image.  The A tensor map has row pitch `channels` and row length kernel_w*channels
 * (rows overlap), and the K loop walks kernel_h row segments shifted by `padded_width` rows.
 * Needs kernel_w*channels % 64 == 0.  act: 0 none, 1 gelu, 2 relu, 3 silu, 5 quick-gelu. */
int vllm_conv_rows_bf16(const void* xpad, long long pad_pixels, int channels, int padded_width, int kernel_h,
                        int kernel_w, const void* weight, int ldw, void* out, int ldo, int out_channels,
                        const void* bias, int act, void* stream);
/* Tile selection for tests and sweeps (process-global): VLLM_GEMM_DEFAULT = the library's choice per launch (128 x 256
 * tiles for dense K-major GEMMs with N >= 2048, else 128 x 128; csrc/gemm.cu), VLLM_GEMM_WIDE_TILE =
 * 128 x 256 tiles, which the scatter GEMM always uses, VLLM_GEMM_NARROW_TILE = 128 x 128 tiles except for the scatter
 * GEMM.  Any other value: VLLM_EINVAL, nothing changes. */
#define VLLM_GEMM_DEFAULT 0
#define VLLM_GEMM_WIDE_TILE 2
#define VLLM_GEMM_NARROW_TILE 3
int vllm_gemm_set_variant(int variant);

/* ---- row-wise norms and RoPE (bf16 in/out, fp32 statistics) ----------------------
 * vllm_rmsnorm_bf16 replaces apex.normalization.FusedRMSNorm forward
 * (apex/csrc/layer_norm_cuda.cpp:436-441 rms_forward_affine; kernel
 * layer_norm_cuda_kernel.cu:353-437) and the python fallbacks InternRMSNorm
 * (internvit/modeling_intern_vit.py:33-44) / InternLM2RMSNorm / LlamaRMSNorm.
 * Rows may be strided (ldx, ldy in elements) so q/k slices of a packed qkv tensor are
 * normalised in place.  cols % 8 == 0, cols <= 16384. */
int vllm_rmsnorm_bf16(const void* x, long long ldx, const void* weight, void* y, long long ldy, long long rows,
                      int cols, float eps, void* stream);
int vllm_layernorm_bf16(const void* x, long long ldx, const void* weight, const void* bias, void* y, long long ldy,
                        long long rows, int cols, float eps, void* stream);
/* LayerNorm followed by exact-erf GELU in one pass (the `LayerNorm -> GELU` tail of the DCNv3 module's depthwise
 * branch, ops_dcnv3/modules/dcnv3.py:252-267). */
int vllm_layernorm_gelu_bf16(const void* x, long long ldx, const void* weight, const void* bias, void* y,
                             long long ldy, long long rows, int cols, float eps, void* stream);
/* LayerNorm with a row gather in the same pass: output row (b, j) = LN(x[b, index[j]]) for j < rows_out, b < batch;
 * index[j] >= rows_in marks a padding slot and yields an all-zero row.  The window partition of a Swin block (HF
 * SwinLayer: layernorm_before -> pad -> roll -> window_partition) as one kernel: `index` is the window-major list of
 * raster positions (visionllm_b200/swin.py), x [batch * rows_in, cols], y [batch * rows_out, cols]. */
int vllm_layernorm_gather_bf16(const void* x, long long ldx, const int64_t* index, long long rows_in, long long rows_out,
                               long long batch, const void* weight, const void* bias, void* y, long long ldy, int cols,
                               float eps, void* stream);
/* y = residual + LayerNorm(x): the post-norm residual of InternImage-H (`x + res_post_norm(dcn(norm(x)))`,
 * grounding_dino/modeling_ov_grounding_dino_mask_dn.py:4866-4868) in one pass. */
int vllm_layernorm_residual_bf16(const void* x, long long ldx, const void* weight, const void* bias,
                                 const void* residual, long long ldr, void* y, long long ldy, long long rows, int cols,
                                 float eps, void* stream);
/* Elementwise companions of the DCNv3 module (ops_dcnv3/modules/dcnv3.py:318-349), fp32:
 * prep: packed[row, :] = [offset (group*taps*2) | mask logits (group*taps) | centre-scale logit (group, only read when
 *       scale != NULL)] with row pitch ld -> contiguous offset, mask = softmax over the taps of each group, scale =
 *       sigmoid(logit); taps = 9 or 25.
 * blend: out = bf16(core * (1 - s) + xproj * s), s = scale[row, channel / group_channels] (scale == NULL: plain cast). */
int vllm_dcnv3_prep_f32(const void* packed, long long ld, void* offset, void* mask, void* scale, long long rows,
                        int group, int taps, void* stream);
int vllm_dcnv3_blend_bf16(const void* core, const void* xproj, const void* scale, void* out, long long rows,
                          int channels, int group_channels, void* stream);
/* Depthwise KxK convolution (K = 3, 5, 7; stride 1, padding K/2) over a channels-last bf16 map x[batch,H,W,C] with
 * fp32 accumulation: the `nn.Conv2d(C, C, k, padding=(k-1)//2, groups=C)` at the head of the DCNv3 module
 * (ops_dcnv3/modules/dcnv3.py:252-259; InternImage-H: k = 5).  weight_taps is the conv weight repacked tap-major
 * [K*K][C] bf16, bias [C] bf16 or NULL, C % 8 == 0. */
int vllm_dwconv_nhwc_bf16(const void* x, const void* weight_taps, const void* bias, void* y, int batch, int height,
                          int width, int channels, int kernel, void* stream);
/* GroupNorm over channels-last rows x[batch, hw, channels] (bf16, fp32 statistics, optional fused ReLU): the
 * nn.GroupNorm(32, d_model) after each Grounding-DINO input projection
 * (grounding_dino/modeling_ov_grounding_dino_mask_dn.py:2085-2110, :2393-2405) and the detectron2
 * Conv2d(norm=GN, activation=relu) blocks of the mask-feature FPN (:2126-2151, :2470-2478).
 * channels/groups % 8 == 0, channels <= 2048.  workspace: vllm_groupnorm_workspace_bytes(batch, groups) bytes of
 * device memory (per-chunk partial sums; combined in a fixed order, so results are run-to-run identical). */
long long vllm_groupnorm_workspace_bytes(int batch, int groups);
/* x is the valid [h, w] corner of a possibly padded grid: pixel (r, c) of image n is read at pixel index
 * n * x_image_pitch + r * x_w_pitch + c (what vllm_conv_rows_bf16 leaves for a 3x3 convolution; a contiguous
 * [batch, hw, channels] input is h = 1, w = x_w_pitch = x_image_pitch = hw); y is the contiguous [batch, h * w, channels]
 * result.  The statistics order does not depend on the pitches, so the result equals copying the corner out first. */
int vllm_groupnorm_nhwc_bf16_grid(const void* x, void* y, const void* gamma, const void* beta, int batch, long long h, long long w,
                                  long long x_w_pitch, long long x_image_pitch, int channels, int groups, float eps, int relu,
                                  void* workspace, long long workspace_bytes, void* stream);
/* FPN top-down step of the Grounding-DINO mask-feature head (modeling_ov_grounding_dino_mask_dn.py:2486-2492):
 * out = lateral + F.interpolate(top, size=(out_h, out_w), mode="bilinear", align_corners=False) over channels-last bf16
 * maps top [batch, in_h, in_w, channels], lateral / out [batch, out_h, out_w, channels] in one pass (ATen's
 * upsample_bilinear2d arithmetic; the interpolated value is rounded to bf16 before the bf16 add, like the torch ops).
 * channels % 8 == 0.  `top` images lie top_image_pitch elements apart (a level slab of the flattened encoder output, read
 * in place; in_h * in_w * channels for a contiguous tensor);
 * out_pad > 0 writes the result into the interior of a caller-zeroed [batch, out_h + 2 pad, out_w + 2 pad, channels] map --
 * the zero-padded input of the 3x3 output convolution that follows (:2493), without a pad copy. */
int vllm_upsample_add_nhwc_bf16_ex(const void* top, long long top_image_pitch, const void* lateral, void* out, int batch, int in_h,
                                   int in_w, int out_h, int out_w, int channels, int out_pad, void* stream);
/* In-place rotate-half RoPE on x[tokens, heads, head_dim] rows with pitch ld; cos/sin
 * [tokens, head_dim] bf16 gathered per position (HF Llama apply_rotary_pos_emb;
 * internlm2/modeling_internlm2.py:218-232). */
int vllm_rope_bf16(void* x, long long ld, const void* cos, const void* sin, long long tokens, int heads,
                   int head_dim, void* stream);

/* ---- fused attention (flash dataflow; scores never reach HBM) ---------------------
 * Replaces flash_attn_varlen_qkvpacked_func (internvit/flash_attention.py:51-54), the
 * FA2 / eager paths of HF Llama and internlm2/modeling_internlm2.py:362-546, and
 * internvit/modeling_intern_vit.py:145-160.  q/k/v: [batch, tokens, heads, head_dim]
 * bf16 views with explicit batch/token pitches in elements (heads contiguous, so a
 * packed qkv GEMM output is read in place); o: [batch, Tq, heads*head_dim] bf16.
 * kv_heads < heads = grouped-query attention.  seqlens (int32[batch], may be NULL):
 * keys >= seqlens[b] are masked (right padding / key_padding_mask); a seqlens[b] >= Tk masks nothing and reads no
 * key past Tk; all query rows are computed.
 * key_mask (uint8 [batch, Tk], may be NULL): 1 = attend, 0 = masked -- an arbitrary key_padding_mask
 * (nn.MultiheadAttention / GroundingDinoBiMultiHeadAttention semantics, inverted).
 * attn_mask (uint8 [batch*heads, Tq, Tk], may be NULL): 1 = attend; exactly the [N*H, L, S] tensor
 * nn.MultiheadAttention receives as `attn_mask` (inverted), indexed by batch*heads + head.
 * attn_bias (fp32 [bias_batches, heads, Tq, Tk], may be NULL): added to the scaled scores before the softmax;
 * batch b reads slab b % bias_batches -- Swin's relative-position bias (+ shifted-window mask, one slab per window
 * of an image; HF modeling_swin.py SwinSelfAttention.forward, used by the reference through AutoBackbone,
 * modeling_ov_grounding_dino_mask_dn.py:471-504).
 * causal != 0: query i sees keys <= i + (Tk - Tq).  head_dim in {32, 64, 128, 256}.
 * scale must be > 0 and finite, else VLLM_EINVAL before anything runs (the wgmma kernel scales after the row max).
 * A query row that can attend no key (seqlens 0, an all-0 key_mask or attn_mask row, a -inf bias row, causal rows
 * i < Tq - Tk) is written as exact zeros.
 * K / V rows that are masked (keys in [seqlens[b], Tk), key_mask 0) must still hold finite values on the default
 * variant: the wgmma kernel multiplies them by P = 0, and NaN * 0 is NaN.  Rows past Tk are never read.
 * workspace (may be NULL): caller-owned scratch of workspace_bytes; when the query side alone cannot fill the
 * GPU (few queries, many keys: GDINO text->vision attention, 80 x 21760) the key axis is split across CTAs and
 * the partials (unnormalised O, running max, sum) are merged by a second kernel.  NULL only turns the split off.
 * n splits use the first batch*heads*n*Tq*(head_dim + 2) floats of it. */
int vllm_attention_bf16(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk,
                        int heads, int kv_heads, int head_dim, long long q_batch_pitch,
                        long long q_token_pitch, long long k_batch_pitch, long long k_token_pitch,
                        long long v_batch_pitch, long long v_token_pitch, long long o_batch_pitch,
                        long long o_token_pitch, const int* seqlens, const unsigned char* key_mask,
                        const unsigned char* attn_mask, const float* attn_bias, int bias_batches, int causal,
                        float scale, void* workspace, long long workspace_bytes, void* stream);
/* Sparse attn_mask (UniPose's keypoint decoder: 50 groups of 1 + 68 queries attend within their group,
 * unipose/modeling_unipose.py:887-917 -- 3450 x 3450 bytes per (image, head), > 95 % blocked): vllm_attention_mask_tiles lists, per
 * (batch*heads, 64-row query block), the ascending ids of the 64-key tiles that hold at least one allowed pair
 * (tile_counts int32 [n_batch_heads, ceil(Tq/64)], tile_lists int32 [n_batch_heads, ceil(Tq/64), ceil(Tk/64)]);
 * vllm_attention_bf16_tiles is vllm_attention_bf16 (non-causal, head_dim 32 / 64 / 128, attn_mask required) walking only those
 * tiles.  A fully blocked tile leaves the online softmax untouched, so the result is bit-identical to the dense walk. */
int vllm_attention_mask_tiles(const unsigned char* attn_mask, long long n_batch_heads, int Tq, int Tk, int* tile_counts,
                              int* tile_lists, void* stream);
int vllm_attention_bf16_tiles(const void* q, const void* k, const void* v, void* o, int batch, int Tq, int Tk,
                              int heads, int kv_heads, int head_dim, long long q_batch_pitch,
                              long long q_token_pitch, long long k_batch_pitch, long long k_token_pitch,
                              long long v_batch_pitch, long long v_token_pitch, long long o_batch_pitch,
                              long long o_token_pitch, const int* seqlens, const unsigned char* key_mask,
                              const unsigned char* attn_mask, float scale, const int* tile_counts,
                              const int* tile_lists, void* stream);
/* Kernel selection for tests and benchmarks (process-global):
 *   VLLM_ATTN_DEFAULT   the first kernel that takes the call: the wgmma kernel (head_dim 128 / 256 without attn_mask /
 *                       attn_bias), the one-warp-per-window Swin kernel (head_dim 32, attn_bias only, no seqlens, not
 *                       causal, Tq == Tk <= 64, kv_heads == heads), else the warp-MMA kernel
 *   VLLM_ATTN_WARP_MMA  switches off the wgmma kernel and the window kernel: every call runs on the warp-MMA kernel
 * Any other value: VLLM_EINVAL, nothing changes. */
#define VLLM_ATTN_DEFAULT 0
#define VLLM_ATTN_WARP_MMA 1
int vllm_attention_set_variant(int variant);
/* Split-KV count for tests (process-global): 0 (the default) lets the library choose; n in 1..64 makes every
 * vllm_attention_bf16 call with a non-NULL workspace split the key axis n ways, on both the wgmma and the warp-MMA kernel
 * and whatever the shape, masks or causal flag.  A NULL workspace, the window kernel and tile-list calls still do not
 * split; a workspace smaller than n partials is VLLM_EINVAL.  Any other n: VLLM_EINVAL, nothing changes. */
int vllm_attention_set_splits(int n);

/* ---- tensor-parallel LLM decoder over peer memory (BASELINE cfg 5, SURVEY 8e) -------
 * The reference runs HF LlamaDecoderLayer unsharded (modeling_visionllmv2.py:724-732); the north-star splits it
 * over the NVSwitch box.  These entry points are the exchange steps of that split, fused with the math either side
 * (visionllm_b200/tp.py is the host mirror; nothing here calls NCCL):
 *   vllm_peer_*            one cudaMalloc'ed, zero-filled exchange buffer per rank, shared through CUDA IPC
 *                          (export = 64-byte handle a rank hands its peers through torch.distributed; open maps a
 *                          peer's buffer and enables P2P access).  These four are setup calls: they allocate and
 *                          synchronise (the only ones in the library that do).
 *   vllm_gemm_bf16_scatter row-parallel o_proj fused with the reduce-scatter PUSH: C = A.B^T, row block d (rows
 *                          [d*rows_per_dst, (d+1)*rows_per_dst)) is stored by the GEMM epilogue directly to dst[d]
 *                          (a peer's receive slot, pitch ldc) tile by tile; each epilogue warp then adds 1 to
 *                          flags[d] with release semantics at system scope: (rows_per_dst/128)*ceil(N/256)*8
 *                          arrivals per destination and call.  rows_per_dst % 128 == 0, N % 64 == 0.
 *   vllm_tp_reduce_norm_bf16  owner side: wait until *wait_flag - wait_target >= 0 (NULL: no wait), x[r,:] +=
 *                          sum_s slots[s][r,:] (fp32, one bf16 rounding, stored in place when n_slots > 0), then
 *                          RMSNorm(x) * weight (the two bf16 roundings of vllm_rmsnorm_bf16) written to dst[0..n_dst)
 *                          at row pitch ld_dst (local MLP input, or every peer's gather buffer = the all-gather),
 *                          then each CTA adds 1 to signal[0..n_signal) (vllm_tp_norm_ctas(rows) CTAs).  cols % 8 == 0, <= 8192.
 *   vllm_tp_wait / vllm_tp_signal  one-thread kernels: spin until a counter reaches target / add to peers' counters
 *                          (the barrier in front of a forward and the wait in front of a GEMM that reads the gather
 *                          buffer through TMA).
 * dst / flags / signal are HOST arrays of device pointers (<= 8 entries). */
int vllm_peer_alloc(void** ptr, size_t bytes);
int vllm_peer_free(void* ptr);
int vllm_peer_handle_bytes(void);
int vllm_peer_export(void* ptr, void* host_handle_out);
int vllm_peer_open(const void* host_handle, void** ptr_out);
int vllm_peer_close(void* ptr);
int vllm_gemm_bf16_scatter(const void* A, int lda, const void* B, int ldb, void* const* dst, void* const* flags,
                           int n_dst, int rows_per_dst, int ldc, int N, int K, void* stream);
int vllm_tp_reduce_norm_bf16(const void* slots, int n_slots, long long slot_stride, void* x, const void* weight,
                             float eps, void* const* dst, int n_dst, long long ld_dst, const void* wait_flag,
                             unsigned wait_target, void* const* signal, int n_signal, int rows, int cols,
                             void* stream);
int vllm_tp_norm_ctas(int rows); /* counter arrivals per destination of one vllm_tp_reduce_norm_bf16 launch */
int vllm_tp_wait(const void* flag, unsigned target, void* stream);
int vllm_tp_signal(void* const* signal, int n_signal, unsigned add, void* stream);

/* ---- Grounding-DINO post-processing (SURVEY 8f rank 3; csrc/postproc.cu) -------------------------------------
 * vllm_det_postprocess_f32 replaces post_process_det_gdino (visionllmv2/eval/eval_det.py:18-56): per image
 * sigmoid(logits[:, :num_classes]) -> top-k over the flattened (query, class) grid -> box_idx = idx // K, label =
 * idx % K (int64) -> gather pred_boxes, cxcywh -> xyxy (util/box_ops.py:16-22), scale by (w, h, w, h).  logits
 * [batch, num_queries, logits_ld] fp32 (only the first num_classes columns of a row are scored), pred_boxes
 * [batch, num_queries, 4] fp32, sizes_hw [batch, 2] fp32 = (img_h, img_w).  Outputs [batch, topk]: scores fp32,
 * topk_indexes / box_idx / labels int64, boxes [batch, topk, 4] fp32.  topk <= min(1024, num_queries*num_classes).
 * Order: probability descending; equal probabilities by ascending flat index (torch leaves ties unspecified). */
int vllm_det_postprocess_f32(const float* logits, const float* pred_boxes, const float* sizes_hw, int batch, int num_queries,
                             int num_classes, int logits_ld, int topk, float* scores, int64_t* topk_indexes,
                             int64_t* box_idx, int64_t* labels, float* boxes, void* stream);
/* vllm_mask_postprocess_f32 replaces the mask branch of post_process_instseg_gdino (eval_det.py:88-99) for ONE image:
 * masks [num_queries, mask_h, mask_w] fp32, box_idx [num_det] int64 -> out [num_det, out_h, out_w] uint8 (0/1) =
 * sigmoid(bilinear(crop(bilinear(masks[box_idx], x mask_stride))[:crop_h, :crop_w] -> (out_h, out_w))) > 0.5, both
 * interpolations with ATen's align_corners=False arithmetic, evaluated analytically (no intermediate tensors). */
int vllm_mask_postprocess_f32(const float* masks, const int64_t* box_idx, int num_det, int mask_h, int mask_w, int mask_stride,
                              int crop_h, int crop_w, int out_h, int out_w, unsigned char* out, void* stream);

/* ---- backward GEMMs (training-side path of BASELINE cfg 5) ----------------------------------------------------
 * C[M, N] = sum_k A(m, k) * B(n, k), bf16 in, fp32 accumulate, bf16 or fp32 out, same wgmma kernel as vllm_gemm_bf16.
 * Each operand is either K-major ([M|N rows, K cols], pitch lda / ldb) or MN-major ([K rows, M|N cols]); MN-major tiles
 * are TMA-loaded as 64 x 64 boxes and fed to wgmma through MN-major shared-memory descriptors, so the backward
 * of y = x W^T (the reference's nn.Linear autograd, torch.nn.functional.linear) needs no transposed copies:
 *   dgrad  dx = dy . W      : A = dy [T, out] K-major,  B = W [out, in]  MN-major,  M = T,   N = in, K = out
 *   wgrad  dW = dy^T . x    : A = dy [T, out] MN-major, B = x [T, in]    MN-major,  M = out, N = in, K = T     */
int vllm_gemm_bf16_tn(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C, int ldc, int M,
                      int N, int K, int out_f32, void* stream);

/* n_batch independent products in one launch (block-diagonal batching): every operand and C are stacks of their
 * n_batch matrices along the row axis.  causal: 0 none; 1 skip output tiles strictly above the diagonal (S = Q K^T,
 * dP = dO V^T); 2 / 3 restrict the K range to where a causal P / dS is non-zero (dV = P^T dO, dK = dS^T Q / dQ = dS K;
 * K is the sequence axis there: K == M is required).
 * M % 256 == 0 (and K % 64 == 0 with MN-major operands) so tiles never straddle two matrices. */
int vllm_gemm_bf16_batched(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C, int ldc,
                           int n_batch, int M, int N, int K, int causal, int out_f32, void* stream);
/* Grouped batching for grouped-query attention (`group` query heads share one KV head; q head i of a batch row belongs to
 * KV head i / group, so "B index = A index / group" and "reduce over `group` consecutive matrices" hold across the batch):
 *   reduce = 0 (broadcast): C and A have n_batch matrices, B has n_batch / group; output matrix i = A_i . B_{i / group}^T.
 *            causal 0 / 1 / 2 / 3 as in vllm_gemm_bf16_batched (S = Q K^T, dP = dO V^T with 1, dQ = dS K with 3).
 *   reduce = 1: A and B have n_batch matrices, C has n_batch / group; output matrix j = sum over g < group of
 *            A_{j group + g} . B_{j group + g}^T, accumulated in fp32 and rounded once (dV = sum_g P_g^T dO_g,
 *            dK = sum_g dS_g^T Q_g).  Both operands MN-major: the reduction is one K axis of group * K rows.  causal 0,
 *            or 2: the K range of every one of the group's segments starts at the tile's first row (K == M required).
 * vllm_gemm_bf16_batched is the group = 1 broadcast.  Returns, with nothing launched:
 *   VLLM_EINVAL        group <= 0, n_batch % group, reduce not 0 / 1, reduce with causal 1 / 3, causal 2 / 3 with K != M,
 *                      and the size / pitch rules of vllm_gemm_bf16_batched;
 *   VLLM_EUNSUPPORTED  reduce with a K-major operand, M % 256, K % 64 with an MN-major operand, a stack over 2^31 rows;
 *   VLLM_EALIGN        bases not 16-byte aligned, pitches not 16-byte multiples. */
int vllm_gemm_bf16_batched_grouped(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, void* C,
                                   int ldc, int n_batch, int group, int reduce, int M, int N, int K, int causal, int out_f32,
                                   void* stream);
/* Row kernels of the training-side path (csrc/train_ops.cu): RMSNorm backward (below, with vllm_rmsnorm_bwd_ws_bf16),
 * SwiGLU forward / backward on the interleaved (gate, up) columns of the gate|up GEMM, the causal
 * softmax / softmax-backward of the materialised attention backward (in place on [n_mat*T, T] bf16 stacks), and the
 * CrossEntropyLoss of modeling_visionllmv2.py:741-757 (fp32 logits, int64 labels, -100 ignored; loss_sum accumulated,
 * dlogits bf16 = (softmax - onehot) / *n_valid). */
/* Layout change of the attention backward (visionllm_b200/train.py): src [batch, tokens, parts, heads, head_dim] bf16 (parts = 3:
 * the packed q | k | v projection rows; 1: dO) -> dst [parts, batch, heads, tokens, head_dim] (every (batch, head) matrix stacked
 * along rows for vllm_gemm_bf16_batched) when to_stacked != 0, the inverse (stacked gradients -> packed d(qkv)) otherwise.
 * One pass of 16-byte vectors; contiguous tensors. */
int vllm_head_stack_bf16(const void* src, void* dst, int batch, int tokens, int parts, int heads, int head_dim,
                         int to_stacked, void* stream);
/* Grouped-query form: packed projection rows [batch, tokens, (nq + 2 nkv) head_dim] bf16 with row pitch ld elements (q heads,
 * then k heads, then v heads) -> Q [batch, nq, tokens, head_dim], K / V [batch, nkv, tokens, head_dim] (contiguous stacks
 * for vllm_gemm_bf16_batched_grouped) when to_stacked != 0, the inverse (stacked gradients -> packed d(qkv)) otherwise.
 * The pitch gap of a packed row is neither read nor written.  nq % nkv != 0 or ld < (nq + 2 nkv) head_dim: VLLM_EINVAL;
 * head_dim % 8 (head_dim < 8 included; only batch * tokens == 0 returns VLLM_OK first): VLLM_EUNSUPPORTED; ld % 8 or a
 * base not 16-byte aligned: VLLM_EALIGN. */
int vllm_head_stack_qkv_bf16(void* packed, long long ld, void* q, void* k, void* v, int batch, int tokens, int nq, int nkv,
                             int head_dim, int to_stacked, void* stream);
/* RMSNorm backward: dx bf16 and dweight fp32, the dweight reduction done through a workspace: every CTA writes its partial
 * column sums to one row of partials [n_partials >= vllm_rmsnorm_bwd_partials(rows), cols] (fp32, 16-byte aligned) and a
 * second kernel sums the rows in order -- deterministic.  dweight is overwritten (no zero-init needed). */
int vllm_rmsnorm_bwd_partials(long long rows);
int vllm_rmsnorm_bwd_ws_bf16(const void* x, long long ldx, const void* weight, const void* dy, long long ldy, void* dx,
                             long long lddx, float* dweight, float* partials, int n_partials, long long rows, int cols,
                             float eps, void* stream);
int vllm_swiglu_fwd_bf16(const void* gate_up, long long ldgu, void* h, long long ldh, long long rows, int inter, void* stream);
int vllm_swiglu_bwd_bf16(const void* gate_up, long long ldgu, const void* dh, long long lddh, void* dgate_up, long long lddgu,
                         long long rows, int inter, void* stream);
int vllm_softmax_causal_bf16(void* s, long long ld, long long n_mat, int T, float scale, void* stream);
int vllm_attn_ds_bf16(const void* p, void* dp, long long ld, long long n_mat, int T, float scale, void* stream);
int vllm_ce_loss_f32(const float* logits, long long ld, const int64_t* labels, const int64_t* n_valid, long long rows, int vocab,
                     float* loss_sum, void* dlogits, long long ldd, void* stream);
/* x [rows, cols] bf16 (row pitch ld) *= *scale in place, the product in fp32 and rounded once; `scale` is one fp32 on the
 * device (the upstream gradient of the loss: CrossEntropyFn.backward scales dlogits by it without a host sync).
 * ld % 8 or a base not 16-byte aligned: VLLM_EALIGN. */
int vllm_scale_rows_bf16(void* x, long long ld, long long rows, int cols, const float* scale, void* stream);
/* Attention backward on right-padded batches of any length (visionllm_b200/train.py): the stacks are padded to tokens_pad
 * rows per (batch, head) matrix (a multiple of 256 for the batched GEMMs).  vllm_head_stack_qkv_pad_bf16 is
 * vllm_head_stack_qkv_bf16 with stacks of tokens_pad rows: rows tokens .. tokens_pad - 1 are written as zeros going to the
 * stacks and are not read coming back; nkv = 0 stacks the nq heads of a plain [batch, tokens, nq head_dim] tensor (dO) into q.
 * Rejections as vllm_head_stack_qkv_bf16 (head_dim < 8 is VLLM_EUNSUPPORTED, not a call that writes nothing), plus
 * tokens_pad < tokens: VLLM_EINVAL.
 * vllm_softmax_causal_len_bf16 is vllm_softmax_causal_bf16 with key lengths lens[n_mat / heads_per_batch] (int32, device):
 * key j of query i is visible iff j <= i and j < lens[m / heads_per_batch]; P = 0 elsewhere (S is not used there), a row
 * with no visible key is all zeros.  n_mat % heads_per_batch: VLLM_EINVAL.  With lens == T it is bit-identical to
 * vllm_softmax_causal_bf16. */
int vllm_head_stack_qkv_pad_bf16(void* packed, long long ld, void* q, void* k, void* v, int batch, int tokens, int tokens_pad,
                                 int nq, int nkv, int head_dim, int to_stacked, void* stream);
int vllm_softmax_causal_len_bf16(void* s, long long ld, long long n_mat, int heads_per_batch, int T, const int* lens,
                                 float scale, void* stream);
/* Backward of the vision-language bridge.  Every parameter gradient is fp32, summed over rows in a fixed order (per-CTA
 * partials in row order, then the partial rows in order, as vllm_rmsnorm_bwd_ws_bf16): run-to-run identical.
 *   vllm_gelu_fwd_bf16   y = gelu(u), exact erf (nn.GELU()), [rows, cols] bf16;
 *   vllm_gelu_bwd_bf16   dx = dy * gelu'(u) from the saved pre-activation u;
 *   vllm_bias_grad_bf16  dbias[c] = sum over rows of dy[r, c];
 *   vllm_layernorm_bwd_wb_bf16  nn.LayerNorm weight / bias gradients, dweight = sum dy * (x - mean) * rstd, dbias = sum dy
 *                        (no dx).  partials [2 n_partials, cols].
 * partials: fp32, 16-byte aligned, n_partials >= vllm_rmsnorm_bwd_partials(rows) rows of cols.  cols % 8: VLLM_EINVAL. */
int vllm_gelu_fwd_bf16(const void* u, long long ldu, void* y, long long ldy, long long rows, int cols, void* stream);
int vllm_gelu_bwd_bf16(const void* u, long long ldu, const void* dy, long long lddy, void* dx, long long lddx, long long rows,
                       int cols, void* stream);
int vllm_bias_grad_bf16(const void* dy, long long ldy, float* dbias, float* partials, int n_partials, long long rows, int cols,
                        void* stream);
int vllm_layernorm_bwd_wb_bf16(const void* x, long long ldx, const void* dy, long long ldy, float* dweight, float* dbias,
                               float* partials, int n_partials, long long rows, int cols, float eps, void* stream);
/* Backward of vllm_assemble_embeds_bf16: the n positions sorted stably by destination row (dest ascending, int32; order[s] the
 * position of entry s) -> d_sources [source_rows, hidden] bf16, every row the fp32 sum, in position order, of the d_embeds
 * rows of the positions naming it, rounded once; rows no position names are exact 0.  The destinations index the
 * concatenation of the sources (token table | [EMB] det table | [EMB] pose table | image features), so one call gives the
 * table gradients and the gather of d(image features) (each feature row is named at most once: an exact copy). */
int vllm_assemble_embeds_bwd_bf16(const int* dest, const int* order, long long n, const void* d_embeds, int hidden,
                                  void* d_sources, long long source_rows, void* stream);
/* Backward of the region encoder (csrc/train_ops.cu).
 *   vllm_layernorm_gelu_bwd_bf16  backward of vllm_layernorm_gelu_bf16 (y = gelu(z), z = (x - mean) * rstd * w + b): the
 *        statistics and z are recomputed with the forward's bits; g = dy * gelu'(z), n = (x - mean) * rstd;
 *        dx = rstd * (w g - mean(w g) - n * mean(w g n)) (bf16, one rounding), dweight = sum g n, dbias = sum g (fp32,
 *        fixed order through partials [2 n_partials, cols], n_partials >= vllm_layernorm_gelu_bwd_partials(rows)).  The
 *        forward's shapes: cols % 8 == 0 and cols <= 16384 (else VLLM_EUNSUPPORTED); rows = 0 zeroes dweight and dbias.
 *   vllm_point_pool_bwd_bf16  backward of the grid_sample point pooling (one-level MSDA sampling of n_points points per
 *        region with weights 1 / 0, a sum and a division by the count) for `levels` feature levels sharing one map:
 *        loc [levels, regions, n_points, 2] fp32 (x, y in [0, 1]), weight [levels, regions, n_points] fp32, counts
 *        [levels, regions] fp32 (the forward's sums of the weights), grad [levels, regions, channels] bf16 ->
 *        d_map [regions, height * width, channels] bf16 = sum_l a_l (x) grad_l / count_l, where a_l is the splat density
 *        of the level's points (their bilinear corner weights times their weight, msda_geom's sampling rule, summed over
 *        the points in index order).  density: fp32 workspace [levels, regions, height * width].  No float atomics:
 *        run-to-run identical.  A level with count 0 adds exact 0. */
long long vllm_layernorm_gelu_bwd_partials(long long rows);
int vllm_layernorm_gelu_bwd_bf16(const void* x, long long ldx, const void* weight, const void* bias, const void* dy,
                                 long long ldy, void* dx, long long lddx, float* dweight, float* dbias, float* partials,
                                 long long n_partials, long long rows, int cols, float eps, void* stream);
int vllm_point_pool_bwd_bf16(const float* loc, const float* weight, const float* counts, int n_points, const void* grad,
                             int levels, int regions, int height, int width, int channels, float* density, void* d_map,
                             void* stream);

/* ---- sequence assembly of VisionLLMv2Model.forward (SURVEY 8f rank 2, 8a-a7/a9; csrc/seqglue.cu) -----------------
 * vllm_seq_index: ONE pass over input_ids [batch, seq_len] (int64, device) producing
 *   new_ids   the ids with [EMB] .. [EMB+num_embs-1] written after every tool token (modeling_visionllmv2.py:447-486,
 *             overwrite form; tool_ids / tool_tables are HOST arrays: table 0 = emb_embeddings_det (det/seg/grd tools),
 *             1 = emb_embeddings_pose),
 *   kind/row  per position where its embedding row comes from: 0 token embedding (row = original id), 1 / 2 the det /
 *             pose [EMB] table (row = j), 3 image feature (row = k-th ViT token of the samples that own <im_patch> tokens,
 *             :582-605; tile_start / tile_count [batch] int32 device arrays give each sample's tile rows, NULL = no images),
 *   emb_pos   [batch, seq_len] int32: positions of the [EMB] tokens of each row in order, emb_count [batch] their number
 *             (:776-787),
 *   status    int32, OR-ed: 1 = a tool token without its pre-placed [EMB] slots (the generation-time insert form, refused),
 *             2 = <im_patch> slots != ViT tokens.  The caller zeroes it first and reads it back.
 * vllm_assemble_embeds_bf16: inputs_embeds [rows, hidden] from kind/row and the four sources (base_embeds, if given,
 * replaces the token-embedding lookup: the caller passed inputs_embeds).  vllm_text_query_gather_bf16: text_query
 * [batch, max_patches, num_embs, hidden] zero padded + masks [batch, max_patches] (uint8).  vllm_gather_rows_bf16:
 * dst[i] = src[idx[i]] (negative idx counts from src_rows).  vllm_pixel_shuffle_rows_bf16: :381-392 + the [:, 1:] CLS
 * slice + optionally the LayerNorm(4C) opening the internvl_mlp bridge in one pass: x = ViT hidden state [tiles,
 * skip_tokens + grid_w*grid_h, C] (pitches ld_tile / ld_token), y = [tiles * grid_w/2 * grid_h/2, 4C]; chunk_order 0 = the
 * reference's pixel_shuffle, 1 = HF SwinPatchMerging's concatenation order (the GDINO backbone's patch merging + its LayerNorm). */
int vllm_seq_index(const int64_t* input_ids, int batch, int seq_len, const int64_t* tool_ids, const int* tool_tables,
                   int num_tools, int64_t emb_token_id, int num_embs, int64_t imp_token_id, const int* tile_start,
                   const int* tile_count, int tokens_per_tile, int64_t* new_ids, unsigned char* kind, int* row, int* emb_pos,
                   int* emb_count, int* status, void* stream);
int vllm_assemble_embeds_bf16(const unsigned char* kind, const int* row, const void* embed_tokens, const void* emb_det,
                              const void* emb_pose, const void* image_features, const void* base_embeds, void* out,
                              long long rows, int hidden, void* stream);
int vllm_text_query_gather_bf16(const void* hidden, const int* emb_pos, const int* emb_count, int batch, int seq_len,
                                int hidden_size, int num_embs, int max_patches, void* text_query, unsigned char* masks,
                                void* stream);
int vllm_gather_rows_bf16(const void* src, long long src_ld, long long src_rows, const int64_t* idx, long long n, int cols,
                          void* dst, void* stream);
int vllm_pixel_shuffle_rows_bf16(const void* x, long long ld_tile, long long ld_token, int skip_tokens, int tiles, int grid_w,
                                 int grid_h, int channels, const void* ln_weight, const void* ln_bias, float eps, void* y,
                                 int chunk_order, void* stream);

/* ---- sine position embeddings of the Grounding-DINO stage (csrc/posembed.cu) ----
 * Replaces the elementwise chains of GroundingDinoSinePositionEmbedding.forward (grounding_dino/
 * modeling_ov_grounding_dino_mask_dn.py:529-564, + the `.to(dtype)` and `+ level_embed` of :2420-2424) and of
 * get_proposal_pos_embed (:1755-1790) by one launch:
 *   out[r, f * nd + d] = (d even ? sin : cos)((feat_f[r * feat_stride] * pre_scale) / dim_t[d]),  f < nfeat <= 4, nd % 8 == 0,
 * fp32 IEEE arithmetic in the reference's order; pre_scale == 0 skips the multiply; dim_t [nd] fp32 is the reference's own
 * temperature ** (2 * (d // 2) / nd) tensor.  out: fp32 [rows, ldo] or (out_bf16) bf16 rounded like `.to(bfloat16)`, then
 * optionally + add_row_bf16 [nfeat * nd] as a bf16 tensor add (fp32 sum, rounded again).  rows_per_batch > 0: output row r is
 * row r % rows_per_batch of slab r / rows_per_batch, slabs out_batch_stride elements apart (one level of a [B, S, C] buffer). */
int vllm_sine_embed_f32(const float* f0, const float* f1, const float* f2, const float* f3, long long feat_stride, int nfeat,
                        float pre_scale, const float* dim_t, int nd, long long rows, void* out, long long ldo, int out_bf16,
                        long long rows_per_batch, long long out_batch_stride, const void* add_row_bf16, void* stream);

#ifdef __cplusplus
}
#endif
#endif
