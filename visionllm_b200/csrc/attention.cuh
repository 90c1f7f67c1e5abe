// What attention.cu and attention_wgmma.cu share: the validated arguments of one attention call, which are also the
// parameters of the warp-MMA kernel, and the entry point of the wgmma kernel.
#pragma once
#include "common.cuh"

struct AttnArgs {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* o;
  long long q_bs, k_bs, v_bs, o_bs;  // batch pitches
  long long q_ts, k_ts, v_ts, o_ts;  // token pitches
  const int* seqlens;
  const unsigned char* key_mask;   // optional [batch, Tk], 1 = attend (arbitrary key_padding_mask)
  const unsigned char* attn_mask;  // optional [batch*heads, Tq, Tk], 1 = attend (nn.MultiheadAttention attn_mask, inverted)
  const float* attn_bias;          // optional additive bias [bias_batches, heads, Tq, Tk] fp32; batch b reads slab b % bias_batches
  int bias_batches;
  int Tq, Tk, heads, kv_heads, causal;
  float scale_log2;
  int n_splits;      // split-KV: CTAs along the key axis per query block (1 = off)
  float* ws;         // workspace [batch*heads*n_splits*Tq][D + 2] fp32 partials (unnormalised O, m, l)
  // Live-tile lists of a sparse attn_mask (vllm_attention_mask_tiles): per (batch*heads, 64-row query block) the ascending
  // ids of the 64-key tiles holding at least one allowed pair.  A fully blocked tile leaves the online softmax untouched
  // (all scores -inf: corr = 1, p = 0), so walking only the live tiles gives bit-identical results.
  const int* tile_counts;   // [batch*heads, q_blocks] or nullptr
  const int* tile_lists;    // [batch*heads, q_blocks, k_tiles]
  int q_blocks, k_tiles;
};

// head_dim 128 / 256 on the wgmma kernel; reads q, k, v, o with their pitches, seqlens, key_mask, causal, scale_log2,
// n_splits and ws (attn_mask, attn_bias and tile lists are not supported).  n_splits > 1: the unnormalised partials go to
// ws and the caller merges them (attention.cu, splitkv_combine_kernel).  VLLM_EUNSUPPORTED: views a TMA descriptor cannot
// express (the caller then uses the warp-MMA kernel).
int vllm_attention_wgmma(const AttnArgs& a, int batch, int head_dim, cudaStream_t st);
