// Process-level helpers of libvllm_b200.so (no kernels here).
#include "common.cuh"

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

extern "C" const char* vllm_version(void) { return "vllm_b200 0.1 sm_90a"; }
