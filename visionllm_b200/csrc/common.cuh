// Shared helpers for the sm_90a kernels behind libvllm_b200.so.
// Everything here is device/host plumbing; no torch types anywhere in csrc/.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

// C-ABI error convention (include/vllm_b200.h): 0 = ok, <0 = argument error,
// >0 = cudaError_t of the failed launch.  The reference only printf()s launch
// errors (mmcv ms_deform_attn_cuda.cu:41-44); we return them.
#define VLLM_OK 0
#define VLLM_EINVAL (-1)
#define VLLM_EUNSUPPORTED (-2)
#define VLLM_EALIGN (-3)

#define VLLM_CHECK_LAUNCH()                          \
  do {                                               \
    cudaError_t _e = cudaGetLastError();             \
    if (_e != cudaSuccess) return (int)_e;           \
  } while (0)

static inline bool vllm_aligned(const void* p, size_t a) {
  return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Raises the dynamic shared-memory limit of kernel `kern` on the current device to at least `bytes`.  The limit is a
// property of the function ON A DEVICE, so what was set is remembered per (device, kernel) and only a larger request
// calls cudaFuncSetAttribute again (runtime.cu).
cudaError_t vllm_smem_optin(const void* kern, int bytes);
template <typename Kern>
static inline cudaError_t vllm_smem_optin(Kern* kern, int bytes) {
  return vllm_smem_optin(reinterpret_cast<const void*>(kern), bytes);
}

// Number of SMs of the current device (cached per process; H100 SXM = 132).
int vllm_num_sms();
