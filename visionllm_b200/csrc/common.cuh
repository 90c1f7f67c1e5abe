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

// Per-device one-time set-up (cudaFuncSetAttribute is a property of the function ON A DEVICE): the flag of the current
// device in a caller-owned array, or nullptr when the device cannot be told (then the caller repeats the set-up).
static inline bool* vllm_device_flag(bool (&flags)[64]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  return &flags[dev];
}

// Number of SMs of the current device (cached per process; H100 SXM = 132).
int vllm_num_sms();
