// common.cuh -- shared helpers for the sm_90a kernels of libupsnet_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/upsnet_b200.h"

#define UPS_CHECK_LAUNCH()                         \
  do {                                             \
    cudaError_t e__ = cudaGetLastError();          \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

#define UPS_CUDA(call)                             \
  do {                                             \
    cudaError_t e__ = (call);                      \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

namespace ups {

constexpr int kNumSMs = 132;  // H100 SXM

// SM count of the device current at the first call, cached for the process; kNumSMs if the query fails
inline int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0, v = kNumSMs;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    sms = v > 0 ? v : kNumSMs;
  }
  return sms;
}

// cudaFuncSetAttribute is per device (and context): remember which devices a kernel has been configured on, so that a
// process driving several GPUs (the reference's thread-per-GPU DataParallel, gpu_nms(device_id)) opts in on each of them.
struct PerDeviceOnce {
  bool done[64] = {};
  bool need() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) d = 0;
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
};

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

__host__ __device__ inline int conv_out_size(int in, int pad, int dil, int k, int stride) {
  return (in + 2 * pad - (dil * (k - 1) + 1)) / stride + 1;
}

// Lays out a caller-owned workspace as consecutive 256-byte-aligned regions, in the order of the take() calls.  On a
// null base it only adds up the size; on the caller's buffer take() also returns each region's address.  So one
// function per entry point both sizes its workspace (for *_workspace_bytes) and carves it.
class WsCarve {
 public:
  explicit WsCarve(void* base) : base_((char*)base) {}
  template <typename T>
  T* take(size_t count) {
    T* p = base_ ? (T*)(base_ + off_) : nullptr;
    off_ = align_up(off_ + count * sizeof(T), 256);
    return p;
  }
  size_t bytes() const { return off_; }

 private:
  char* base_;
  size_t off_ = 0;
};

}  // namespace ups
