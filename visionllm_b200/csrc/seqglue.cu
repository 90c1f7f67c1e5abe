// Host-side sequence assembly of VisionLLMv2Model.forward as kernels (SURVEY 8f rank 2 + 8a-a7): pure integer index
// work and row copies, exact by construction.
//
//   seq_index_kernel        visionllmv2/model/modeling_visionllmv2.py:426-468 ([EMB] ids / embeddings overwritten after
//                           det / seg / grd / pose tool tokens), :582-605 (k-th <im_patch> slot of the flattened batch
//                           takes the k-th ViT token of the samples that have image tokens) and the position list of
//                           :776-787 ([EMB] hidden states -> text_query), all from ONE pass over input_ids: writes the
//                           rewritten ids and, per position, where its embedding row comes from.
//   assemble_embeds_kernel  builds inputs_embeds [B*L, C] in one pass from {embed_tokens, emb_embeddings_det / _pose,
//                           image features} (the reference: embedding lookup, then python loops of torch.cat per tool
//                           token, then a masked index_put).
//   text_query_kernel       :776-787: text_query [B, mx, num_embs, C] (zero padded) and text_query_masks [B, mx].
//   gather_rows_kernel      dst[i] = src[idx[i]] (lm_head on requested rows only).
//   pixel_shuffle_ln_kernel :381-392 + :574-579: space-to-depth x2 of the ViT patch tokens (two view/permute/contiguous
//                           copies in the reference, plus the [:, 1:] CLS slice) folded into the LayerNorm that opens the
//                           `internvl_mlp` bridge (or a plain one-pass gather for the other bridges): output row
//                           (n, a, b) = [x(2a, 2b) | x(2a, 2b+1) | x(2a+1, 2b) | x(2a+1, 2b+1)], x indexed (row, column) of the
//                           tile's token grid -- the projector GEMM's A operand is produced directly.
#include "rows.cuh"

namespace {

constexpr int SEQ_THREADS = 1024;
constexpr int MAX_TOOLS = 8;
constexpr int MAX_SAMPLES = 1024;

struct SeqTools {
  long long id[MAX_TOOLS];     // tool token ids (unused entries: -1)
  int table[MAX_TOOLS];        // 0: emb_embeddings_det, 1: emb_embeddings_pose
};

// kind: 0 token embedding (row = original id), 1 det table (row = j), 2 pose table (row = j), 3 image feature (row = k)
__global__ void __launch_bounds__(SEQ_THREADS)
seq_index_kernel(const int64_t* __restrict__ ids, int B, int L, const __grid_constant__ SeqTools tools, long long emb_id,
                 int num_embs, long long imp_id, const int* __restrict__ tile_start, const int* __restrict__ tile_count,
                 int tokens_per_tile, int64_t* __restrict__ new_ids, unsigned char* __restrict__ kind,
                 int* __restrict__ row, int* __restrict__ emb_pos, int* __restrict__ emb_count, int* __restrict__ status) {
  __shared__ int s_scan[SEQ_THREADS / 32];
  __shared__ int s_base;
  __shared__ int s_imp[MAX_SAMPLES];          // <im_patch> tokens per sample
  __shared__ int s_rows_before[MAX_SAMPLES + 1];
  const int tid = threadIdx.x;
  const long long n = (long long)B * L;
  int bad = 0;
  // pass 1: copy ids, token-embedding default
  for (long long i = tid; i < n; i += SEQ_THREADS) {
    const long long v = ids[i];
    new_ids[i] = v;
    kind[i] = 0;
    row[i] = (int)v;
  }
  for (int b = tid; b < B; b += SEQ_THREADS) s_imp[b] = 0;
  __syncthreads();
  // pass 2: [EMB] overwrite after tool tokens (det-class tools first, then pose: mv2.py:447-486 order)
  for (int tbl = 0; tbl < 2; ++tbl) {
    for (long long i = tid; i < n; i += SEQ_THREADS) {
      const long long v = ids[i];
      bool is_tool = false;
#pragma unroll
      for (int t = 0; t < MAX_TOOLS; ++t) is_tool |= (tools.id[t] >= 0 && tools.table[t] == tbl && v == tools.id[t]);
      if (!is_tool) continue;
      const int p = (int)(i % L);
      for (int j = 0; j < num_embs; ++j) {
        const int pj = p + 1 + j;
        if (pj >= L) { bad |= 1; break; }
        const long long slot = ids[i + 1 + j];
        if (slot < emb_id || slot >= emb_id + num_embs) { bad |= 1; break; }   // generation-time insert form: refused
        new_ids[i + 1 + j] = emb_id + j;
        kind[i + 1 + j] = (unsigned char)(1 + tbl);
        row[i + 1 + j] = j;
      }
    }
    __syncthreads();
  }
  // pass 3: per-sample <im_patch> counts (on the rewritten ids)
  if (imp_id >= 0) {
    for (long long i = tid; i < n; i += SEQ_THREADS)
      if (new_ids[i] == imp_id) atomicAdd(&s_imp[(int)(i / L)], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int acc = 0;
    for (int b = 0; b < B; ++b) {                       // rows of image_features[has_image] before sample b's tiles
      s_rows_before[b] = acc;
      if (s_imp[b] > 0 && tile_count) acc += tile_count[b] * tokens_per_tile;
    }
    s_rows_before[B] = acc;
    s_base = 0;
  }
  __syncthreads();
  // pass 4: k-th <im_patch> slot in flat order -> k-th included feature row; [EMB] rank within its row
  int total_imp = 0;
  for (int b = 0; b < B; ++b) total_imp += s_imp[b];
  if (imp_id >= 0 && tile_count) {
    if (total_imp != s_rows_before[B]) bad |= 2;
    for (long long base = 0; base < n; base += SEQ_THREADS) {
      const long long i = base + tid;
      const bool sel = i < n && new_ids[i] == imp_id;
      const unsigned bal = __ballot_sync(0xffffffffu, sel);
      if ((tid & 31) == 0) s_scan[tid >> 5] = __popc(bal);
      __syncthreads();
      if (sel) {
        int k = s_base;
        for (int w = 0; w < (tid >> 5); ++w) k += s_scan[w];
        k += __popc(bal & ((1u << (tid & 31)) - 1u));
        // k-th row of the concatenation of the included samples' tile rows
        int b = 0;
        while (b + 1 < B && !(s_imp[b] > 0 && k < s_rows_before[b + 1])) ++b;
        if (k < s_rows_before[B]) {
          kind[i] = 3;
          row[i] = tile_start[b] * tokens_per_tile + (k - s_rows_before[b]);
        }
      }
      __syncthreads();
      if (tid == 0) {
        int tot = 0;
        for (int w = 0; w < SEQ_THREADS / 32; ++w) tot += s_scan[w];
        s_base += tot;
      }
      __syncthreads();
    }
  }
  // pass 5: [EMB] positions per row, in order (one warp per row)
  const int warp = tid >> 5, lane = tid & 31;
  for (int b = warp; b < B; b += SEQ_THREADS / 32) {
    int cnt = 0;
    for (int p0 = 0; p0 < L; p0 += 32) {
      const int p = p0 + lane;
      const long long v = p < L ? new_ids[(long long)b * L + p] : -1;
      const bool is_emb = v >= emb_id && v < emb_id + num_embs;
      const unsigned bal = __ballot_sync(0xffffffffu, is_emb);
      if (is_emb) emb_pos[(long long)b * L + cnt + __popc(bal & ((1u << lane) - 1u))] = p;
      cnt += __popc(bal);
    }
    if (lane == 0) emb_count[b] = cnt;
  }
  if (bad) atomicOr(status, bad);
}

__global__ void __launch_bounds__(256)
assemble_embeds_kernel(const unsigned char* __restrict__ kind, const int* __restrict__ row,
                       const __nv_bfloat16* __restrict__ embed, const __nv_bfloat16* __restrict__ det,
                       const __nv_bfloat16* __restrict__ pose, const __nv_bfloat16* __restrict__ image,
                       const __nv_bfloat16* __restrict__ base, __nv_bfloat16* __restrict__ out, long long n, int C) {
  const int nvec = C / 8;
  const int vpr = blockDim.x;                          // one CTA walks rows; threads stride over the row's vectors
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    const int k = kind[i];
    const __nv_bfloat16* src;
    if (k == 0) src = base ? base + i * C : embed + (long long)row[i] * C;   // caller-provided inputs_embeds or the lookup
    else if (k == 1) src = det + (long long)row[i] * C;
    else if (k == 2) src = pose + (long long)row[i] * C;
    else src = image + (long long)row[i] * C;
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(out + i * C);
    for (int v = threadIdx.x; v < nvec; v += vpr) d[v] = __ldg(s + v);
  }
}

__global__ void __launch_bounds__(256)
text_query_kernel(const __nv_bfloat16* __restrict__ hidden, const int* __restrict__ emb_pos,
                  const int* __restrict__ emb_count, int B, int L, int C, int num_embs, int mx,
                  __nv_bfloat16* __restrict__ tq, unsigned char* __restrict__ tm) {
  const int slots = mx * num_embs;
  const int nvec = C / 8;
  for (long long s = blockIdx.x; s < (long long)B * slots; s += gridDim.x) {
    const int b = (int)(s / slots), r = (int)(s - (long long)b * slots);
    const int usable = (emb_count[b] / num_embs) * num_embs;
    const bool ok = r < usable;
    uint4* d = reinterpret_cast<uint4*>(tq + s * C);
    if (ok) {
      const uint4* src = reinterpret_cast<const uint4*>(hidden + ((long long)b * L + emb_pos[(long long)b * L + r]) * C);
      for (int v = threadIdx.x; v < nvec; v += blockDim.x) d[v] = __ldg(src + v);
    } else {
      for (int v = threadIdx.x; v < nvec; v += blockDim.x) d[v] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (threadIdx.x == 0 && r % num_embs == 0) tm[(long long)b * mx + r / num_embs] = ok ? 1 : 0;
  }
}

__global__ void __launch_bounds__(256)
gather_rows_kernel(const __nv_bfloat16* __restrict__ src, long long ld, const int64_t* __restrict__ idx, long long n,
                   long long src_rows, int C, __nv_bfloat16* __restrict__ dst) {
  const int nvec = C / 8;
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    long long r = idx[i];
    if (r < 0) r += src_rows;                            // python-style negative indices
    const uint4* s = reinterpret_cast<const uint4*>(src + r * ld);
    uint4* d = reinterpret_cast<uint4*>(dst + i * C);
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) d[v] = __ldg(s + v);
  }
}

// Narrow rows (the Swin window-reverse gather: C = 96 ... 768): one 16-byte vector per thread, flat over (row, vector), so a
// warp writes 512 contiguous bytes and reads whole source rows; the CTA-per-row kernel above would keep 12 of 256 threads busy.
__global__ void __launch_bounds__(256)
gather_rows_flat_kernel(const __nv_bfloat16* __restrict__ src, long long ld, const int64_t* __restrict__ idx, long long n,
                        long long src_rows, int nvec, __nv_bfloat16* __restrict__ dst) {
  const long long total = n * nvec;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (long long)gridDim.x * blockDim.x) {
    const long long i = v / nvec;
    const int c = (int)(v - i * nvec);
    long long r = idx[i];
    if (r < 0) r += src_rows;
    reinterpret_cast<uint4*>(dst)[v] = __ldg(reinterpret_cast<const uint4*>(src + r * ld) + c);
  }
}

// One CTA (256 threads) per output row of 4*C columns; VPT 16-byte vectors per thread stay in registers between the
// statistics and the scaling pass.  LN: with LayerNorm(4C) (weight, bias), the steps of norm_rows_kernel<1>.  A separate
// kernel rather than a row source of norm_rows_kernel: folded in, its short rows (C = 96 ... 384) ran 16% slower.
template <int VPT, bool LN>
__global__ void __launch_bounds__(256)
pixel_shuffle_ln_kernel(const __nv_bfloat16* __restrict__ x, long long ld_tile, long long ld_token, int skip, int gw, int gh,
                        int C, const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ bias, float eps,
                        __nv_bfloat16* __restrict__ y, int order) {
  __shared__ float sh[8];
  const int ow = gw / 2, oh = gh / 2;
  const long long r = blockIdx.x;                        // (tile, a, b)
  const int tile = (int)(r / (ow * oh)), ab = (int)(r - (long long)tile * ow * oh);
  const int a = ab / oh, b = ab - a * oh;
  const int cvec = C / 8, nvec = 4 * cvec;
  const __nv_bfloat16* xt = x + tile * ld_tile + (long long)skip * ld_token;
  uint4 reg[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * 256;
    reg[i] = make_uint4(0u, 0u, 0u, 0u);
    if (v < nvec) {
      const int chunk = v / cvec, cv = v - chunk * cvec;
      // order 0 (pixel shuffle, mv2.py:381-392): chunk = (dy, dx) = (chunk >> 1, chunk & 1);
      // order 1 (Swin patch merging, HF SwinPatchMerging: cat[x(0::2,0::2), x(1::2,0::2), x(0::2,1::2), x(1::2,1::2)]): (chunk & 1, chunk >> 1)
      const int dy = order ? (chunk & 1) : (chunk >> 1), dx = order ? (chunk >> 1) : (chunk & 1);
      const long long tok = (long long)(2 * a + dy) * gh + (2 * b + dx);
      reg[i] = __ldg(reinterpret_cast<const uint4*>(xt + tok * ld_token) + cv);
    }
  }
  float2 st;
  if (LN) st = ln_stats<VPT, 256>(reg, 4 * C, eps, sh);
  uint4* yr = reinterpret_cast<uint4*>(y + r * 4 * C);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * 256;
    if (v < nvec) {
      if (LN) {
        float o[8];
        ln_apply(reg[i], w, bias, v, st, o);
        yr[v] = pack8(o);
      } else {
        yr[v] = reg[i];
      }
    }
  }
}

}  // namespace

extern "C" {

int vllm_seq_index(const int64_t* input_ids, int batch, int seq_len, const int64_t* tool_ids, const int* tool_tables,
                   int num_tools, int64_t emb_token_id, int num_embs, int64_t imp_token_id, const int* tile_start,
                   const int* tile_count, int tokens_per_tile, int64_t* new_ids, unsigned char* kind, int* row, int* emb_pos,
                   int* emb_count, int* status, void* stream) {
  if (batch < 0 || seq_len < 0 || num_tools < 0 || num_tools > MAX_TOOLS || num_embs <= 0) return VLLM_EINVAL;
  if (batch > MAX_SAMPLES) return VLLM_EUNSUPPORTED;
  if ((long long)batch * seq_len == 0) return VLLM_OK;
  if (!input_ids || !new_ids || !kind || !row || !emb_pos || !emb_count || !status) return VLLM_EINVAL;
  SeqTools t;
  for (int i = 0; i < MAX_TOOLS; ++i) {
    t.id[i] = i < num_tools ? tool_ids[i] : -1;           // host arrays
    t.table[i] = i < num_tools ? tool_tables[i] : 0;
  }
  seq_index_kernel<<<1, SEQ_THREADS, 0, (cudaStream_t)stream>>>(input_ids, batch, seq_len, t, emb_token_id, num_embs,
                                                               imp_token_id, tile_start, tile_count, tokens_per_tile, new_ids,
                                                               kind, row, emb_pos, emb_count, status);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_assemble_embeds_bf16(const unsigned char* kind, const int* row, const void* embed_tokens, const void* emb_det,
                              const void* emb_pose, const void* image_features, const void* base_embeds, void* out,
                              long long rows, int hidden, void* stream) {
  if (rows < 0 || hidden <= 0 || hidden % 8) return VLLM_EINVAL;
  if (rows == 0) return VLLM_OK;
  if (!kind || !row || !out || (!embed_tokens && !base_embeds)) return VLLM_EINVAL;
  long long blocks = rows < (long long)vllm_num_sms() * 16 ? rows : (long long)vllm_num_sms() * 16;
  assemble_embeds_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      kind, row, (const __nv_bfloat16*)embed_tokens, (const __nv_bfloat16*)emb_det, (const __nv_bfloat16*)emb_pose,
      (const __nv_bfloat16*)image_features, (const __nv_bfloat16*)base_embeds, (__nv_bfloat16*)out, rows, hidden);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_text_query_gather_bf16(const void* hidden, const int* emb_pos, const int* emb_count, int batch, int seq_len,
                                int hidden_size, int num_embs, int max_patches, void* text_query, unsigned char* masks,
                                void* stream) {
  if (batch < 0 || seq_len < 0 || hidden_size <= 0 || hidden_size % 8 || num_embs <= 0 || max_patches < 0) return VLLM_EINVAL;
  const long long slots = (long long)batch * max_patches * num_embs;
  if (slots == 0) return VLLM_OK;
  if (!hidden || !emb_pos || !emb_count || !text_query || !masks) return VLLM_EINVAL;
  long long blocks = slots < (long long)vllm_num_sms() * 16 ? slots : (long long)vllm_num_sms() * 16;
  text_query_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)hidden, emb_pos, emb_count, batch,
                                                                        seq_len, hidden_size, num_embs, max_patches,
                                                                        (__nv_bfloat16*)text_query, masks);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_gather_rows_bf16(const void* src, long long src_ld, long long src_rows, const int64_t* idx, long long n, int cols,
                          void* dst, void* stream) {
  if (n < 0 || cols <= 0 || cols % 8 || src_ld < cols) return VLLM_EINVAL;
  if (n == 0) return VLLM_OK;
  if (!src || !idx || !dst) return VLLM_EINVAL;
  if (src_ld % 8 || !vllm_aligned(src, 16) || !vllm_aligned(dst, 16)) return VLLM_EALIGN;
  const int nvec = cols / 8;
  if (nvec < 128) {
    long long blocks = (n * nvec + 255) / 256;
    const long long cap = (long long)vllm_num_sms() * 32;
    if (blocks > cap) blocks = cap;
    gather_rows_flat_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, src_ld, idx, n, src_rows,
                                                                               nvec, (__nv_bfloat16*)dst);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  }
  long long blocks = n < (long long)vllm_num_sms() * 16 ? n : (long long)vllm_num_sms() * 16;
  gather_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, src_ld, idx, n, src_rows, cols,
                                                                         (__nv_bfloat16*)dst);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_pixel_shuffle_rows_bf16(const void* x, long long ld_tile, long long ld_token, int skip_tokens, int tiles, int grid_w,
                                 int grid_h, int channels, const void* ln_weight, const void* ln_bias, float eps, void* y,
                                 int chunk_order, void* stream) {
  if (tiles < 0 || grid_w <= 0 || grid_h <= 0 || (grid_w & 1) || (grid_h & 1) || channels <= 0 || channels % 8) return VLLM_EINVAL;
  if (chunk_order != 0 && chunk_order != 1) return VLLM_EINVAL;
  if (tiles == 0) return VLLM_OK;
  if (!x || !y || ((ln_weight == nullptr) != (ln_bias == nullptr))) return VLLM_EINVAL;
  if (ld_token % 8 || ld_tile % 8 || !vllm_aligned(x, 16) || !vllm_aligned(y, 16)) return VLLM_EALIGN;
  const int nvec = 4 * channels / 8;
  const long long rows = (long long)tiles * (grid_w / 2) * (grid_h / 2);
  if (rows > 2147483647LL) return VLLM_EUNSUPPORTED;
  const bool ln = ln_weight != nullptr;
  return with_vpt<256, 2, 4, 8>(nvec, [&](auto vpt, auto) -> int {
    constexpr int VPT = decltype(vpt)::value;
    if (ln)
      pixel_shuffle_ln_kernel<VPT, true><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
          (const __nv_bfloat16*)x, ld_tile, ld_token, skip_tokens, grid_w, grid_h, channels, (const __nv_bfloat16*)ln_weight,
          (const __nv_bfloat16*)ln_bias, eps, (__nv_bfloat16*)y, chunk_order);
    else
      pixel_shuffle_ln_kernel<VPT, false><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
          (const __nv_bfloat16*)x, ld_tile, ld_token, skip_tokens, grid_w, grid_h, channels, nullptr, nullptr, eps,
          (__nv_bfloat16*)y, chunk_order);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

}  // extern "C"
