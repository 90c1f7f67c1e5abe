// Peer-memory plumbing and the fused "reduce + residual + RMSNorm + push" kernel of the tensor-parallel LLM path
// (BASELINE cfg 5 / SURVEY.md 8e: the LLM decoder split over the GPUs of one NVSwitch box).
//
// The reference has no tensor parallelism (its Llama is HF's, sharded only by DeepSpeed ZeRO, SURVEY 2.3); what is
// replaced here is the pair "row-parallel o_proj -> all-reduce -> +residual -> RMSNorm" a Megatron-style split of
// HF LlamaDecoderLayer would run as four kernels and one NCCL call.  Layout of the exchange (visionllm_b200/tp.py):
//
//   * every rank owns R = M / W consecutive token rows of the residual stream (sequence-parallel between the
//     attention blocks) and nq / W attention heads;
//   * o_proj: each rank's GEMM epilogue stores its partial [M, H] tile by tile straight into the OWNER's receive
//     slots over NVLink (vllm_gemm_bf16_scatter, gemm.cu) and bumps the owner's arrival counter per tile;
//   * tp_reduce_norm_kernel (here) on the owner: waits for the counter, sums the W partial slots in fp32, adds the
//     residual row, stores the new residual, applies RMSNorm (same two bf16 roundings as vllm_rmsnorm_bf16) and
//     stores the normalised row either locally (input of the sequence-parallel MLP) or into EVERY peer's gather
//     buffer (the all-gather in front of the next QKV GEMM), then bumps the peers' counters.
//
// One reduce-scatter (inside the GEMM epilogue) and one all-gather (inside the norm kernel) per layer = the volume
// of a single all-reduce, with no NCCL call on the data path.  Counters only grow (epoch * arrivals-per-epoch), so
// no reset traffic; comparisons are wrap-safe.
//
// Memory model: writers issue plain stores to peer memory, then fence.acq_rel.sys, then red.release.sys on the
// counter; the reader spins with ld.acquire.sys and reads the slots with ld.global.cg (L2 is the coherence point of
// device memory written by peers; L1 is bypassed).
#include "rows.cuh"
#include <string.h>

#define TP_MAX_PEERS 8

namespace {

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// A peer that never arrives (crashed rank, protocol bug) must not hang the GPU: after TP_SPIN_TIMEOUT_NS the waiter
// traps, which surfaces as a CUDA error on the host instead of a dead box.
#define TP_SPIN_TIMEOUT_NS 20000000000ull
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void spin_until(const uint32_t* flag, uint32_t target) {
  if ((int32_t)(ld_acquire_sys(flag) - target) >= 0) return;
  const unsigned long long t0 = global_ns();
  while ((int32_t)(ld_acquire_sys(flag) - target) < 0) {
    __nanosleep(64);
    if (global_ns() - t0 > TP_SPIN_TIMEOUT_NS) __trap();
  }
}
__device__ __forceinline__ uint4 ld_cg_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
struct TpNormArgs {
  const __nv_bfloat16* slots; int n_slots; long long slot_stride;   // [n_slots][rows][cols] partial sums (local)
  __nv_bfloat16* x;                                                  // [rows, cols] residual stream (local, in place)
  const __nv_bfloat16* w; float eps;                                 // RMSNorm weight
  __nv_bfloat16* dst[TP_MAX_PEERS]; int n_dst; long long ld_dst;     // normalised rows go to every dst (row-offset applied)
  const uint32_t* wait_flag; uint32_t wait_target;                   // arrival counter of the slots (null: no wait)
  uint32_t* signal[TP_MAX_PEERS]; int n_signal;                      // counters bumped once per CTA after the pushes
  int rows, cols;
};

constexpr int TPN_THREADS = 256;

// A CTA walks rows blockIdx.x, blockIdx.x + gridDim.x, ...; thread t owns 16-byte vectors t, t+256, ... of a row
// (VPT of them, cols <= 8 * 256 * VPT).  One wait at the start and ONE fence + counter bump per CTA at the end (a
// system-scope fence per row costs more than the row itself), so a push arrives as gridDim.x counts per source.
template <int VPT>
__global__ void __launch_bounds__(TPN_THREADS)
tp_reduce_norm_kernel(const TpNormArgs a) {
  __shared__ float sh[2][TPN_THREADS / 32];
  const int nvec = a.cols / 8;
  if (a.wait_flag) {
    if (threadIdx.x == 0) spin_until(a.wait_flag, a.wait_target);
    __syncthreads();
  }
  int it = 0;
  for (int row = blockIdx.x; row < a.rows; row += gridDim.x, it ^= 1) {
    uint4 reg[VPT];
    __nv_bfloat16* xr = a.x + (size_t)row * a.cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * TPN_THREADS;
      reg[i] = make_uint4(0u, 0u, 0u, 0u);
      if (v < nvec) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int s = 0; s < a.n_slots; ++s) {
          float f[8];
          unpack8(ld_cg_u4(a.slots + (size_t)s * a.slot_stride + (size_t)row * a.cols + 8 * v), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
        float f[8];
        unpack8(*(reinterpret_cast<const uint4*>(xr) + v), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
        reg[i] = pack8(acc);                            // the new residual, rounded once to bf16 like a GEMM epilogue;
        if (a.n_slots > 0) *(reinterpret_cast<uint4*>(xr) + v) = reg[i];   // RMSNorm sees the stored (rounded) value
      }
    }
    // double-buffered sh: one barrier per row
    const float inv = rms_rstd<VPT, TPN_THREADS, false>(reg, a.cols, a.eps, sh[it]);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * TPN_THREADS;
      if (v < nvec) {
        const uint4 pk = rms_apply(reg[i], a.w, v, inv);
        for (int d = 0; d < a.n_dst; ++d)
          *(reinterpret_cast<uint4*>(a.dst[d] + (size_t)row * a.ld_dst) + v) = pk;
      }
    }
  }
  if (a.n_signal > 0) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < a.n_signal) red_release_sys(a.signal[threadIdx.x], 1u);
  }
}

__global__ void tp_wait_kernel(const uint32_t* flag, uint32_t target) { spin_until(flag, target); }

struct TpSignalArgs { uint32_t* signal[TP_MAX_PEERS]; int n; uint32_t add; };
__global__ void tp_signal_all_kernel(const TpSignalArgs a) {
  __threadfence_system();
  if (threadIdx.x < a.n) red_release_sys(a.signal[threadIdx.x], a.add);
}

}  // namespace

extern "C" {

// ---- peer allocations (cudaMalloc + legacy CUDA IPC; one handle per rank) ----
int vllm_peer_alloc(void** ptr, size_t bytes) {
  if (!ptr || bytes == 0) return VLLM_EINVAL;
  cudaError_t e = cudaMalloc(ptr, bytes);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemset(*ptr, 0, bytes);
  if (e != cudaSuccess) return (int)e;
  e = cudaDeviceSynchronize();
  return e == cudaSuccess ? VLLM_OK : (int)e;
}
int vllm_peer_free(void* ptr) {
  if (!ptr) return VLLM_OK;
  cudaError_t e = cudaFree(ptr);
  return e == cudaSuccess ? VLLM_OK : (int)e;
}
int vllm_peer_handle_bytes(void) { return (int)sizeof(cudaIpcMemHandle_t); }
int vllm_peer_export(void* ptr, void* handle_out) {
  if (!ptr || !handle_out) return VLLM_EINVAL;
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
  if (e != cudaSuccess) return (int)e;
  memcpy(handle_out, &h, sizeof(h));
  return VLLM_OK;
}
int vllm_peer_open(const void* handle, void** ptr_out) {
  if (!handle || !ptr_out) return VLLM_EINVAL;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  cudaError_t e = cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? VLLM_OK : (int)e;
}
int vllm_peer_close(void* ptr) {
  if (!ptr) return VLLM_OK;
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  return e == cudaSuccess ? VLLM_OK : (int)e;
}

// CTAs (= counter arrivals per destination) of one vllm_tp_reduce_norm_bf16 launch over `rows` rows; every rank of a
// box has the same SM count, so producer and consumer compute the same number.
int vllm_tp_norm_ctas(int rows) {
  const int cap = vllm_num_sms() * 4;
  return rows < cap ? (rows > 0 ? rows : 1) : cap;
}

int vllm_tp_reduce_norm_bf16(const void* slots, int n_slots, long long slot_stride, void* x, const void* weight,
                             float eps, void* const* dst, int n_dst, long long ld_dst, const void* wait_flag,
                             unsigned wait_target, void* const* signal, int n_signal, int rows, int cols,
                             void* stream) {
  if (rows < 0 || cols <= 0 || n_slots < 0 || n_dst < 0 || n_signal < 0) return VLLM_EINVAL;
  if (n_slots > TP_MAX_PEERS || n_dst > TP_MAX_PEERS || n_signal > TP_MAX_PEERS) return VLLM_EUNSUPPORTED;
  if (rows == 0) return VLLM_OK;
  if (!x || !weight || (n_slots && !slots) || (n_dst && !dst) || (n_signal && !signal)) return VLLM_EINVAL;
  if (cols % 8 || cols > 8 * TPN_THREADS * 4 || (n_dst && ld_dst % 8)) return VLLM_EUNSUPPORTED;
  if (!vllm_aligned(x, 16) || !vllm_aligned(weight, 16) || (n_slots && (!vllm_aligned(slots, 16) || slot_stride % 8)))
    return VLLM_EALIGN;
  TpNormArgs a{};
  a.slots = (const __nv_bfloat16*)slots; a.n_slots = n_slots; a.slot_stride = slot_stride;
  a.x = (__nv_bfloat16*)x; a.w = (const __nv_bfloat16*)weight; a.eps = eps;
  for (int d = 0; d < n_dst; ++d) {
    if (!dst[d] || !vllm_aligned(dst[d], 16)) return VLLM_EALIGN;
    a.dst[d] = (__nv_bfloat16*)dst[d];
  }
  a.n_dst = n_dst; a.ld_dst = ld_dst;
  a.wait_flag = (const uint32_t*)wait_flag; a.wait_target = wait_target;
  for (int d = 0; d < n_signal; ++d) {
    if (!signal[d]) return VLLM_EINVAL;
    a.signal[d] = (uint32_t*)signal[d];
  }
  a.n_signal = n_signal; a.rows = rows; a.cols = cols;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = vllm_tp_norm_ctas(rows);
  return with_vpt<TPN_THREADS, 1, 2, 4>(cols / 8, [&](auto vpt, auto) {
    tp_reduce_norm_kernel<decltype(vpt)::value><<<grid, TPN_THREADS, 0, st>>>(a);
    VLLM_CHECK_LAUNCH();
    return VLLM_OK;
  });
}

int vllm_tp_wait(const void* flag, unsigned target, void* stream) {
  if (!flag) return VLLM_EINVAL;
  tp_wait_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((const uint32_t*)flag, target);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

int vllm_tp_signal(void* const* signal, int n_signal, unsigned add, void* stream) {
  if (n_signal < 0 || n_signal > TP_MAX_PEERS || (n_signal && !signal)) return VLLM_EINVAL;
  if (n_signal == 0) return VLLM_OK;
  TpSignalArgs a{};
  for (int d = 0; d < n_signal; ++d) {
    if (!signal[d]) return VLLM_EINVAL;
    a.signal[d] = (uint32_t*)signal[d];
  }
  a.n = n_signal; a.add = add;
  tp_signal_all_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  VLLM_CHECK_LAUNCH();
  return VLLM_OK;
}

}  // extern "C"
