// Process-level helpers of libvllm_b200.so (no kernels here).
#include "common.cuh"
#include <map>
#include <mutex>
#include <utility>

int vllm_num_sms() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    sms[dev] = n;
  }
  return sms[dev];
}

cudaError_t vllm_smem_optin(const void* kern, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> limit;   // (device, kernel) -> bytes set there
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  int& set = limit[{dev, kern}];
  if (set >= bytes) return cudaSuccess;
  const cudaError_t r = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (r == cudaSuccess) set = bytes;
  return r;
}

extern "C" const char* vllm_version(void) { return "vllm_b200 0.1 sm_90a"; }
